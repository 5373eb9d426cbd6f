// scrolly_maze.cu — fused step kernel for examples/scrolly_maze.py.
//
// One launch = Engine.play() for every env (engine.py:583-639): the three
// update groups [['#'], ['a','b','c','P'], ['@']] (scrolly_maze.py:241), the
// Plot consultation, and the final z-ordered render 'abc@#P' (:242).
//
// The two intermediate renders of the reference (one per update group,
// engine.py:735) are never materialised: the only board cells the entities
// read between groups are the <= 9 neighbours of a MazeWalker, tested against
// impassable = '#', and in z-order 'abc@#P' a cell shows '#' iff the wall
// curtain covers it and the (previously rendered) player is not standing on
// it.
//
// Memory schedule (one warp per env, everything staged through shared memory):
//   1. records (sprites/drapes/plot, 64 words) -> smem with two coalesced loads;
//      only the fields this game uses are pulled into registers;
//   2. group 0 ('#' MazeDrape) is pure register arithmetic and fixes BOTH
//      final window corners (the '@' drape can only obey an order, never issue
//      one: by the time it runs, the player's permit is already for frame+1);
//   3. the patch trip, one job and at most two words per lane, every load issued before
//      any is used: each of the 4 walkers' 5x5 patch of wall bits as one word of the
//      level's wall-neighbourhood table (covers every cell any _check_motion of this step
//      can consult, wherever the scroll order moves the walker first), the 3x3 patch of
//      coin bits around the player, and on the delta path the coin and backdrop rows
//      around each sprite;
//   4. once those bits are in, cp.async of the backdrop tile and of the two windows of
//      the bit-packed patterns (4 words per row, one 16-byte copy from the row-blocked
//      copies of the bound patterns, see "Row-blocked windows") -> smem, no registers
//      held; groups 1 and 2 run on registers + shuffles of the patch bits while the
//      copies fly;
//   5. each lane shifts whole window rows once into one word per 16-cell board
//      segment (wall16 << 16 | coin16); the paint loop then composes 16-byte
//      segments from smem (prmt with a 256-entry selector table) and streams them
//      out with uint4 stores; records go back with two coalesced stores.
// So a step costs two dependent round trips (records, then the patch rows) before the
// bulk copies start.  In a full wave (32 warps per SM) those trips, not a warp's own
// arithmetic, set the step's length: with the copies issued first, every warp's 6 KB of
// copies queued in front of them (DESIGN.md section 5, tools/step_phases.py).
//
// Not built: several envs per warp.  Packing E envs into a warp divides the warp-uniform
// game logic per env by E, and leaves a 4096-env launch with the warps per SM of a
// 4096 / E-env launch today.  The delta-path kernel at 1024 and 2048 envs (8 and 16 warps
// per SM; an optimistic bound for E = 4 and 2, with fewer loads per warp) steps in 7.89
// and 7.30 us against 8.26 at 4096 (H100 SXM, 700 W, tools/step_sweep.py; DESIGN.md
// section 5): at most ~12 %, and E = 4 would not beat E = 2.  The wave's length is not
// issue contention between the SM's warps.  (An earlier GPU's A/B of two envs per warp
// was slower too, but for another reason: before delta rendering, halving the lanes
// doubled the staging and paint loops on each warp's chain.)
//
// Residency on H100 (64x64 board): 64 registers x 128 threads allow 8 blocks of the
// 65 536 registers, and 6400 B of dynamic shared memory per warp (25 KB per block) + 2 KB
// of static selector tables + the 1 KB per-block reserve = 28 KB per block allow 8 of the
// SM's 228 KB (static_assert below).  8 blocks = 32 warps per SM (__launch_bounds__(128,
// 8)) = 4224 envs per wave on 132 SMs, so a 4096-env launch is one wave.  At 7 blocks (72
// registers, segment words in a buffer of their own) it was 1.11 waves: 17.0 us per
// 4096-env step against 15.0 us at 8 (H100 SXM, 700 W; tools/step_sweep.py and
// DESIGN.md section 5).  Holding 64 registers without spills is why the '@' drape and the
// coin count are read from the records only in group 2, and the records' global addresses
// are recomputed where they are used.
//
// Sprite order P,a,b,c (indices 0..3); drape order '#','@' (0, 1).
// Registers: patroller aux0 = moving_east; P aux0/aux1 = scroll permit mask /
// permit frame; '@' aux0/aux1 = board cell of a coin already removed from the
// pattern but still on the (not yet refreshed) curtain, or -1; '@' aux2 = dirty-group
// mask of the env's coin pattern (below); plot aux0 = coins left in the pattern.
//
// Coin groups: every env owns a complete copy of its level's coin pattern
// (d_pattern[1]), and it differs from the level's template (d_pattern_init[1], shared
// by all envs of the level and so served from L2) only in the rows of coins picked up
// this episode.  Bit k of '@' aux2 set means rows [k g, (k + 1) g) of the env's pattern
// may differ from the template; bit k clear means they are equal.  The step reads a
// clean group's rows from the template instead of the env's copy (the coin window and
// the coin patch rows), a pick-up sets its group's bit, and an auto-reset restart
// copies back only the dirty groups (the reloaded record brings the mask back to 0).
// A host that writes an env's coin pattern directly sets that env's aux2 to -1.
//
// Delta rendering: with the example's margins a window scrolls only when the player comes
// within 2 rows or 3 columns of the board's edge, which the bench workload never did in
// 19 200 env-steps (tools/scroll_census.py).  Then the new board differs from the last one
// in at most the sprites' old and new cells, the old and new stale coin and a picked-up
// coin.  Each env's render key (StepParams::render_key, built by derive(), invalid after
// every pcl_bind_state) records what its last render was drawn from: the frame, the board
// buffer's epoch (StepParams::board_epoch), both corners, each sprite's visible cell, the
// stale coin and the coin mask.  A step that is no restart or reset, whose records match
// the key, whose mask is not -1 and whose windows stay where they are after group 0 takes
// the delta path: it stages nothing; in the patch trip, spare loads fetch the 3x3 coin
// bits and backdrop bytes around each sprite's start cell (the 5x5 wall patches cover the
// walls); after group 2 one lane per candidate cell composes its final value and stores
// that byte.  If '@' then issues its own order, or a candidate lies outside every loaded
// neighbourhood, the warp stages the full paint's copies there and paints in full.  Every
// path that paints writes the key; frozen envs touch neither board nor key.  A host that
// writes into a step's board buffer passes another buffer or binds again (include/pcl.h).
#include <algorithm>
#include <new>

#include "pcl_device.cuh"
#include "pcl_kernels.cuh"
#include "pcl_crop.cuh"

namespace pcl {

namespace {

constexpr int kS = 4;
constexpr int kWarpsPerBlock = 4;
constexpr int kRecWords = 64;     // 4 sprites * 8 + 2 drapes * 8 + plot 16

__device__ __forceinline__ int action_to_motion(int a) {   // scrolly_maze.py:262-271
  // actions 0..4 = N S W E stay (motion codes 0 4 6 2 8), anything else = no motion:
  // one nibble per action in a constant instead of a chain of selects
  constexpr unsigned kTable = (PCL_M_N) | (PCL_M_S << 4) | (PCL_M_W << 8) | (PCL_M_E << 12) |
                              (PCL_M_STAY << 16);
  return (unsigned)a < 5u ? (int)((kTable >> (4 * a)) & 15u) : PCL_M_NONE;
}

__device__ __forceinline__ void cp_async8(void* smem, const void* gmem) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" ::
               "r"((uint32_t)__cvta_generic_to_shared(smem)), "l"(gmem));
}
// 16 bytes through L1, for data every warp of an SM reads (the selector table): the SM's
// warps hit its L1 instead of all sending the same lines to L2 (cp_async16 bypasses L1).
__device__ __forceinline__ void cp_async16_l1(void* smem, const void* gmem) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 16;\n" ::
               "r"((uint32_t)__cvta_generic_to_shared(smem)), "l"(gmem));
}

// The patch trip's loads, with an L2 policy that evicts their lines last: a full paint
// streams ~10 KB per env through L2 (staged tile and windows, the board), which would
// otherwise push the wall-neighbourhood table out and put a DRAM round trip on the step.
__device__ __forceinline__ uint64_t l2_evict_last() {
  uint64_t policy;
  asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(policy));
  return policy;
}
__device__ __forceinline__ uint32_t ld_keep(const uint32_t* p, uint64_t policy) {
  uint32_t v;
  asm volatile("ld.global.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(policy) : "memory");
  return v;
}

// A 64-cell window row starts at bit corner_c of its pattern row; the four words
// from the even word at or below corner_c >> 5 always cover it (<= 31 + 32 + 64
// bits), and pattern rows are 8-byte aligned (pattern_words is even), so a row is
// staged with two 8-byte cp.async into a 16-byte smem slot.

// Pattern rows per bit of the coin dirty-group mask: g = 2^s rows, s the smallest shift
// with 32 g >= PH, so that 32 bits cover every pattern row (g = 8 at 129 rows).
__device__ __forceinline__ int coin_group_shift(int PH) {
  return 32 - __clz((PH - 1) >> 5);
}

// prmt.b32 without __byte_perm's selector masking (the table holds nibbles 0..5).
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
  uint32_t d;
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(sel));
  return d;
}

// Words staged per window row: a W-cell window row starts at bit corner_c of its
// pattern row; from the even word at or below corner_c >> 5 it spans at most
// 63 + W bits.  4 words (two 8-byte cp.async, one 16-byte slot) up to W = 64, 6 or 8
// beyond (drapes.py:293-376 puts no limit on the board width).  The narrow path always
// stages and reads 4 words per row, so a one-column board is floored at 4 too (at
// W = 1, 63 + W bits fit in 2 words).  check_spec checks pattern_words by the same rule.
__host__ __device__ constexpr int window_words(int W) {
  return W < 2 ? 4 : 2 * ((63 + W + 63) / 64);
}

// The 4-word fast paths of staging and segment building: a board row is at most 4
// segments (pitch >= W, so W <= 64 too).
__host__ __device__ constexpr bool narrow_board(int pitch) { return pitch <= 64; }

// Render key (see "Delta rendering"): words per env in the handle's key array, and the
// words in use.  Word i is key_word(rec, i, epoch) of the records the board was drawn from:
// words 0..7 are record words (frame, both corners, the stale coin cell, the coin mask),
// word 8 the board epoch, words 9..12 each sprite's cell row * pitch + col, or -1 if hidden.
constexpr int kKeyStride = 16;
enum { kKeyRecWords = 8, kKeyEpoch = 8, kKeySprites = 9, kKeyWords = kKeySprites + kS };
// Record offsets of key words 0..7, one byte each.
constexpr uint64_t kKeyRec =
    (uint64_t)(48 + PCL_P_FRAME) | (uint64_t)(32 + PCL_D_CORNER_R) << 8 |
    (uint64_t)(32 + PCL_D_CORNER_C) << 16 | (uint64_t)(40 + PCL_D_CORNER_R) << 24 |
    (uint64_t)(40 + PCL_D_CORNER_C) << 32 | (uint64_t)(40 + PCL_D_AUX0) << 40 |
    (uint64_t)(40 + PCL_D_AUX1) << 48 | (uint64_t)(40 + PCL_D_AUX2) << 56;
static_assert(kKeyWords <= kKeyStride, "the render key outgrew its slot");

// Delta rendering's scratch words, in the (then idle) staging area of the warp: the 5x5
// wall words of the walkers, the 3x3 coin rows and backdrop rows around each sprite's
// start cell, and what the last render drew from the records.
enum {
  kNbWall = 0,                     // 4 words: walker s's 5x5 wall word at s
  kNbCoin = 32,                    // 12 words: 3 coin bits per row, sprite s row k at 3 s + k
  kNbBackdrop = 44,                // 12 words: 3 backdrop bytes per row, likewise (kNbCoin + 12)
  kNbStart = 56,                   // 4 words per sprite: vrow, vcol, and row, col (-1: hidden)
  kNbStale = kNbStart + 4 * kS,    // 2 words: the stale coin cell (AUX0, AUX1)
  kNbWords = (kNbStale + 2 + 3) & ~3   // whole 16-byte units: warp regions stay 16-byte aligned
};
static_assert(kNbBackdrop == kNbCoin + 12, "the patch trip stores coin and backdrop rows as one run");

__host__ __device__ constexpr size_t staging_bytes(int H, int W, int pitch) {
  // backdrop tile, two window rows of window_words(W) per board row, and one word per
  // 16-cell segment.  On narrow boards the segment words (pitch / 16 <= 4 per row) take
  // the place of the wall window rows (4 words per row), which are dead by then.
  return (size_t)H * pitch + 2 * ((((size_t)H * window_words(W) * 4) + 15) & ~(size_t)15) +
         (narrow_board(pitch) ? 0 : (((size_t)H * (pitch >> 2) + 15) & ~(size_t)15));
}

__host__ __device__ constexpr size_t warp_smem_bytes(int H, int W, int pitch) {
  // records, then the staging area; the delta path's scratch (kNbWords) reuses the
  // staging area, which tiny boards pad to its size.
  return kRecWords * 4 + (staging_bytes(H, W, pitch) > (size_t)kNbWords * 4
                             ? staging_bytes(H, W, pitch) : (size_t)kNbWords * 4);
}

// Programmatic dependent launch: let the next kernel of the stream begin its
// launch/prologue while this one runs, and wait for everything earlier in the
// stream before touching global memory.
__device__ __forceinline__ void pdl_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
__device__ __forceinline__ void pdl_wait_prior_grids() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
}

// ---- Block chaining (StepParams::chain, block_sync) ------------------------------------
// Step t + 1 of an env reads only what step t of the same env wrote, static level data and
// inputs written before the chain of step launches began.  So when the stream's previous
// kernel is a step launch of this library that shares no per-env memory with this one
// (CHAIN_FOLLOWS, set by api.cu), a block need not wait in griddepcontrol.wait for every
// block of the previous grid to finish and flush: block b waits only for block b of its own
// handle's previous launch.  Freed SM slots then take the next launch's blocks at once, and
// the wave's slowest warps no longer hold every SM idle.  Two counters per block, begin[b]
// and end[b]: the handle's launches whose block b has begun, and those whose block b ended.
//   CHAIN_FOLLOWS  entry: thread 0 takes begun = begin[b]++ with an atomic, waits until
//                  end[b] == begun (block b of every earlier launch of the handle that
//                  counts is done) and acquires what those blocks wrote; the block barrier
//                  passes that on to every warp.  Only then does the block call
//                  launch_dependents.
//   CHAIN_HEAD     the full wait, and the counters kept as above: a step launch whose
//                  predecessor is a step launch it may not chain to (the first of a run, or
//                  a batch sharing memory with the one before).  Thread 0's atomic is issued
//                  before the wait and overlaps it; the block calls launch_dependents after
//                  the wait, so a chained successor starts only once every kernel before
//                  this one has completed.
//   CHAIN_NONE     the kernel as before chaining (launch_dependents at entry, the full
//                  wait), counters untouched: every other launch, such as eager pcl_step or
//                  a step after another kernel.  api.cu never chains a launch to it: the
//                  next step launch is then CHAIN_HEAD at most.
//   exit (HEAD, FOLLOWS): after a block barrier (every warp has left the step: frozen,
//                  ragged-block and early-return warps too), thread 0 stores end[b] =
//                  begun + 1 with st.release.gpu.
// No deadlock: a chained launch may start only once every block of the previous one has
// called launch_dependents, so once each of them is resident and past its own wait; by
// induction the same holds back to the CHAIN_HEAD launch that began the chain, whose wait
// saw every kernel before it complete.  A spinning block
// therefore waits on blocks that are resident and need nothing more to finish, and never
// holds a slot one of them still needs.  The full griddepcontrol.wait waits for every
// prerequisite grid in flight, chained ones included, so a launch after a chain needs
// nothing more.  Inputs another kernel wrote before the chain (actions, the reset mask) are
// read from L2 (ld.global.cg), never from a line an SM's L1 kept from before.
__device__ __forceinline__ uint32_t ld_relaxed_gpu(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_acquire_gpu(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_gpu(uint32_t* p, uint32_t v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}

// Selector table of the paint loop (see the kernel): 256 x u16, built at compile
// time and pulled into shared memory with one cp.async per lane by each warp that paints.
struct SelTable { uint16_t v[256]; };
constexpr SelTable make_sel_table() {
  SelTable t = {};
  for (int idx = 0; idx < 256; ++idx) {
    unsigned sel = 0;
    for (int k = 0; k < 4; ++k) {
      const unsigned nib = ((idx >> (4 + k)) & 1) ? 5u : ((idx >> k) & 1) ? 4u : (unsigned)k;
      sel |= nib << (4 * k);
    }
    t.v[idx] = (uint16_t)sel;
  }
  return t;
}
__device__ __align__(16) const SelTable g_sel = make_sel_table();

// Phase stamps (build with -DPCL_STEP_STAMPS; read by tools/step_phases.py through
// pcl_step_stamps): lane 0 of each warp stores the low 32 bits of its SM's cycle counter
// at each phase boundary, and of %globaltimer (ns) at entry and exit, to
// g_stamps[env].  Differences of these 32-bit stamps, taken modulo 2^32, are exact.
// Without the switch PCL_STAMP expands to nothing and the kernel is the production one.
// The stamp build also fits 64 registers, with a 4-byte spill since the path word;
// tools/step_phases.py reports its step time beside the production build's.
// Slot kStPath names the path the warp took (kPath*), so the tool can tell which path's
// warps end a launch.
#ifdef PCL_STEP_STAMPS
constexpr int kStampEnvs = 8192;
enum {
  kStEntry, kStPrior, kStRecords, kStPatch, kStGroup2, kStWait, kStPatched, kStPaint, kStEnd,
  kStTimeIn, kStTimeOut, kStPath, kStampWords
};
enum { kPathDelta, kPathDeltaPickup, kPathFellBack, kPathFull, kPathRestart };
__device__ uint32_t g_stamps[kStampEnvs][kStampWords];
__device__ __forceinline__ uint32_t global_ns() {
  uint32_t t;
  asm volatile("mov.u32 %0, %%globaltimer_lo;" : "=r"(t));
  return t;
}
// The env index is re-read at every stamp, so no stamp address stays live in between.
__device__ __forceinline__ void stamp(int k, uint32_t v) {
  uint32_t tid, cta;
  asm volatile("mov.u32 %0, %%tid.x;" : "=r"(tid));
  asm volatile("mov.u32 %0, %%ctaid.x;" : "=r"(cta));
  const uint32_t e = cta * kWarpsPerBlock + (tid >> 5);
  if ((tid & 31) == 0 && e < (uint32_t)kStampEnvs) g_stamps[e][k] = v;
}
#define PCL_STAMP(k) stamp(k, (uint32_t)clock())
#define PCL_STAMP_TIME(k) stamp(k, global_ns())
#define PCL_STAMP_PATH(v) stamp(kStPath, (uint32_t)(v))
#else
#define PCL_STAMP(k) do {} while (0)
#define PCL_STAMP_TIME(k) do {} while (0)
#define PCL_STAMP_PATH(v) do {} while (0)
#endif

// The most dynamic shared memory a block may ask for: the block budget less the kernel's
// 2 KB of static selector tables.  check_spec accepts a spec only if its block fits, so
// an accepted spec always launches.
constexpr size_t kMaxDynamicSmem = kMaxBlockSmem - kWarpsPerBlock * sizeof(SelTable);

// 8 blocks per SM (__launch_bounds__ below) on a 64x64 board: a block's dynamic shared
// memory, its per-warp selector tables and the 1 KB the SM reserves per block fit 8 times
// in the H100's 228 KB.
static_assert(8 * (kWarpsPerBlock * (warp_smem_bytes(64, 64, 64) + sizeof(SelTable)) + 1024) <=
                  228 * 1024,
              "a 64x64 scrolly_maze block no longer fits 8 times per SM");
static_assert(warp_smem_bytes(1, 1, 16) == kRecWords * 4 + kNbWords * 4,
              "delta rendering's scratch must fit a warp's region on the smallest board");
static_assert(kMaxDynamicSmem == kMaxBlockSmem - 2048,
              "kMaxDynamicSmem must leave room for the static selector tables");

// 3x3 "blocked" mask (bit (dr+1)*3 + dc+1, sprites.py:495-507) around the virtual
// position (vrow, vcol) of a walker whose 5x5 wall patch `field` is centred on
// (r0, c0): a cell blocks iff it is on the board, the wall curtain covers it and the
// player is not painted over it (z-order ... '#' 'P').  Pure per-lane arithmetic.
__device__ __forceinline__ unsigned blocked3x3(int vrow, int vcol, int r0, int c0, unsigned field,
                                               int H, int W, bool p_vis, int p_row, int p_col) {
  const int br = vrow - r0 + 1, bc = vcol - c0 + 1;    // 3x3 origin inside the 5x5: 0..2
  if ((unsigned)br > 2u || (unsigned)bc > 2u) return 0u;   // cannot happen (|order|, |move| <= 1)
  unsigned colmask = 0;
#pragma unroll
  for (int i = 0; i < 3; ++i) colmask |= ((unsigned)(vcol - 1 + i) < (unsigned)W ? 1u : 0u) << i;
  unsigned blk = 0;
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    unsigned bits = (field >> ((br + j) * 5 + bc)) & colmask;
    if ((unsigned)(vrow - 1 + j) >= (unsigned)H) bits = 0;
    blk |= bits << (3 * j);
  }
  const int dr = p_row - vrow + 1, dc = p_col - vcol + 1;
  if (p_vis && (unsigned)dr <= 2u && (unsigned)dc <= 2u) blk &= ~(1u << (dr * 3 + dc));
  return blk;
}

// All eight motions of sprites.py:479-546 at once: bit m set = motion code m is
// legal (N NE E SE S SW W NW), plus STAY.
__device__ __forceinline__ int legal_motions(unsigned b) {
  const unsigned nw = b & 1u, n = (b >> 1) & 1u, ne = (b >> 2) & 1u, w = (b >> 3) & 1u,
                 e = (b >> 5) & 1u, sw = (b >> 6) & 1u, s = (b >> 7) & 1u, se = (b >> 8) & 1u;
  const unsigned blocked = n | ((ne | (n & e)) << 1) | (e << 2) | ((se | (s & e)) << 3) |
                           (s << 4) | ((sw | (s & w)) << 5) | (w << 6) | ((nw | (n & w)) << 7);
  return (int)((~blocked & 0xffu) | (1u << PCL_M_STAY));
}

// drapes.py:487-659 `_maybe_move` when the player is the only possible egocentric
// participant (validated in pcl_create): same decisions as pcl::scrolly_move.
__device__ __forceinline__ void scrolly_move_p(Drape& d, const ScrollyCfg& cfg, int motion,
                                               Plot& plot, int p_row, int p_col, int p_permit,
                                               int p_permit_frame) {
  if (d.last_frame < plot.frame) {
    d.last_frame = plot.frame;
    d.pre_r = d.corner_r; d.pre_c = d.corner_c;
  }
  const int dr = motion_dr(motion), dc = motion_dc(motion);
  if (plot.order_frame == plot.frame) {          // obey an existing order :513-535
    if (dr != plot.order_r && dc != plot.order_c) plot.error |= PCL_ENV_ERR_ORDER_MISMATCH;
    d.corner_r += plot.order_r; d.corner_c += plot.order_c;
    return;
  }
  if (motion == PCL_M_STAY) return;
  const bool ego = plot.ego_mask & 1;
  const bool possible = !ego || (p_permit_frame == plot.frame && ((p_permit >> motion) & 1));
  int orr, occ;
  if (!cfg.have_margins) {                       // :598-623
    if (!possible) return;
    const int nr = d.corner_r + dr, nc = d.corner_c + dc;
    orr = (0 <= nr && nr <= cfg.limit_r) ? dr : 0;
    occ = (0 <= nc && nc <= cfg.limit_c) ? dc : 0;
  } else {                                       // :625-687
    if (!ego) return;
    const int nr = p_row + dr, nc = p_col + dc;  // TRUE position
    const bool want_v = (p_row > nr && nr <= cfg.m_north) || (p_row < nr && nr >= cfg.m_south);
    const bool want_h = (p_col > nc && nc <= cfg.m_west) || (p_col < nc && nc >= cfg.m_east);
    if (!(want_v || want_h)) return;
    orr = want_v ? dr : 0; occ = want_h ? dc : 0;
    const int cr = d.corner_r + orr, cc = d.corner_c + occ;
    if (!((0 <= cr && cr <= cfg.limit_r) && (0 <= cc && cc <= cfg.limit_c)) || !possible) return;
  }
  d.corner_r += orr; d.corner_c += occ;
  plot.order_r = orr; plot.order_c = occ; plot.order_frame = plot.frame;
}

// The env's own coin pattern, its level's template and its level's wall pattern.  All are
// recomputed from the launch parameters where they are used: at 64 registers, no pointer
// to any of them stays live through the step.
// The index of the env's static level data.  Re-read where it is used after the patch
// trip: at 64 registers the 64-bit index is not held through groups 1 and 2 either.
__device__ __forceinline__ int64_t level_of(const StepParams& p, int env) {
  return p.st.d_level ? p.st.d_level[env] : env;
}
__device__ __forceinline__ const uint32_t* level_walls(const StepParams& p, int64_t lvl) {
  return p.st.d_pattern[0] + lvl * p.st.pattern_bstride[0];
}
__device__ __forceinline__ uint32_t* env_coins(const StepParams& p, int env) {
  return p.st.d_pattern[1] + (int64_t)env * p.st.pattern_bstride[1];
}
__device__ __forceinline__ const uint32_t* level_coins(const StepParams& p, int64_t lvl) {
  return p.st.d_pattern_init[1] + lvl * p.st.pattern_init_bstride[1];
}

// Word i of the render key of records `rec` (kKey*), for a board of row pitch `pitch` in
// the buffer of epoch `epoch`.  Lane i computes word i: no branch on i.
__device__ __forceinline__ int32_t key_word(const int32_t* rec, int i, uint32_t epoch, int pitch) {
  const int32_t r = rec[i < kKeyRecWords ? (int)((kKeyRec >> (8 * i)) & 0xffu) : 0];
  const int32_t* q = rec + min(max(i - kKeySprites, 0), kS - 1) * PCL_SPRITE_WORDS;
  const int32_t cell = q[PCL_S_FLAGS] & 1 ? q[PCL_S_ROW] * pitch + q[PCL_S_COL] : -1;
  return i < kKeyRecWords ? r : i == kKeyEpoch ? (int32_t)epoch : cell;
}

// One warp's env of one step; scrolly_maze_step runs it between the block's entry and exit
// of "Block chaining".  Every return leaves the step for that warp only.
__device__ __forceinline__ void step_env(const StepParams& p) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  // Byte-permute selectors for 4 cells at once: index = wall nibble << 4 | coin
  // nibble; selector nibble k picks byte 5 ('#') if wall_k, else byte 4 ('@') if
  // coin_k, else byte k of the backdrop word (z-order ... '@' '#' ...).
  // One copy per WARP: a warp then needs no block barrier before it paints (warps of a
  // block leave at different points: ragged tail, frozen envs).  Only a warp that paints
  // in full copies it, with its staging copies (stage() below).
  __shared__ __align__(16) uint16_t s_sel_all[kWarpsPerBlock][256];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  uint16_t* s_sel = s_sel_all[warp];
  const int env = blockIdx.x * kWarpsPerBlock + warp;
  const bool live = env < p.B;
  const int H = p.H, W = p.W, PWW = p.PWW;
  const int pitch = p.pitch;
  const int nw = window_words(W);            // staged words per window row (4 for W <= 64)

  uint8_t* my = smem_raw + warp * warp_smem_bytes(H, W, pitch);
  int32_t* rec = reinterpret_cast<int32_t*>(my);
  uint8_t* s_bd = my + kRecWords * 4;
  uint32_t* s_wall = reinterpret_cast<uint32_t*>(s_bd + (size_t)H * pitch);
  uint32_t* s_coin = s_wall + ((H * nw + 3) & ~3);
  // An attached cropper reads its corner state at the very end: start that line's trip
  // from DRAM now (a hint, no register held).
  if (p.has_cropper && p.cropper.state && live && lane == 0)
    asm volatile("prefetch.global.L2 [%0];" :: "l"(p.cropper.state + (int64_t)env * 4));
  if (!live) return;           // ragged last block
  const int64_t lvl = level_of(p, env);     // index of static level data

  // The env's action word does not depend on the records either: issue its load now,
  // beside theirs, instead of one memory round trip later (it is only USED if the env
  // neither restarts nor is frozen).
  int action = p.mode == MODE_STEP ? __ldcg(p.actions + (int64_t)env * p.actions_per_env)
                                   : PCL_ACTION_NONE;
  // The render key, in the same trip as the records.
  const int32_t key = lane < kKeyWords ? p.render_key[(int64_t)env * kKeyStride + lane] : 0;
  // ---- 1. records -> smem (coalesced) ------------------------------------
  rec[lane] = p.st.d_sprites[(int64_t)env * kS * PCL_SPRITE_WORDS + lane];
  rec[32 + lane] = lane < 16 ? p.st.d_drapes[(int64_t)env * 2 * PCL_DRAPE_WORDS + lane]
                             : p.st.d_plot[(int64_t)env * PCL_PLOT_WORDS + lane - 16];
  __syncwarp();
  PCL_STAMP(kStRecords);
  // The decision of pcl::env_run, written out: through the helper this kernel compiles
  // to a few more instructions here, and its H100 step measured ~0.9% slower.
  const int was_over = rec[48 + PCL_P_GAME_OVER];
  bool restart;
  bool frozen = false;
  if (p.mode == MODE_RESET) {
    restart = (p.env_mask == nullptr) || (__ldcg(p.env_mask + env) != 0);
    frozen = !restart;
  } else {
    restart = was_over && p.auto_reset;
    frozen = was_over && !p.auto_reset;
  }
  if (frozen) return;                        // warp-uniform
  // The board in d_board was drawn from these very records (see "Delta rendering").
  const bool key_ok = __all_sync(PCL_FULL, lane >= kKeyWords ||
                                               key == key_word(rec, lane, p.board_epoch, pitch));
  if (restart) {
    const PlotCarry carry = plot_carry(rec + 48, true);
    // Groups of the coin pattern to restore, read before the record is reloaded: the
    // dirty ones at an auto-reset, every one at the host's reset (which so repairs any
    // pattern).
    const unsigned dirty = p.mode == MODE_RESET ? ~0u
                                                : (unsigned)rec[32 + PCL_DRAPE_WORDS + PCL_D_AUX2];
    __syncwarp();
    const int32_t* si = p.st.d_sprites_init + lvl * p.st.sprites_init_bstride;
    const int32_t* di = p.st.d_drapes_init + lvl * p.st.drapes_init_bstride;
    const int32_t* pi = p.st.d_plot_init + lvl * p.st.plot_init_bstride;
    rec[lane] = __ldg(si + lane);
    rec[32 + lane] = lane < 16 ? __ldg(di + lane) : __ldg(pi + lane - 16);
    // Fresh coins: restore the mutable pattern (one Engine per episode); the reloaded
    // record's mask is 0.
    const uint32_t* src = level_coins(p, lvl);
    const int n = p.PH * PWW, gw = PWW << coin_group_shift(p.PH);   // words per group
    for (unsigned m = dirty; m != 0u; m &= m - 1u) {
      const int lo = (__ffs(m) - 1) * gw, hi = min(lo + gw, n);
      for (int i = lo + lane; i < hi; i += 32) env_coins(p, env)[i] = __ldg(src + i);
    }
    __syncwarp();
    if (lane == 0) store_carry(rec + 48, carry);
    __syncwarp();
    action = PCL_ACTION_NONE;
  }

  // ---- registers: the drapes / plot / player fields every lane needs, plus ONE
  // walker per lane (lane & 3: P, a, b, c) for the SIMT part of group 1 ---------
  const int me = lane & 3;
  Sprite mine = load_sprite(rec + me * PCL_SPRITE_WORDS);
  // The player as every lane sees it (previous render + permits).
  const int p_row = rec[PCL_S_ROW], p_col = rec[PCL_S_COL];
  const int p_vrow = rec[PCL_S_VROW], p_vcol = rec[PCL_S_VCOL];
  const bool p_vis = rec[PCL_S_FLAGS] & 1;
  const int p_permit = rec[PCL_S_AUX0], p_permit_frame = rec[PCL_S_AUX1];
  // The '@' drape and the plot's coin count stay in the records until group 2: they
  // are not held in registers through group 1.
  const int32_t* rec_coins = rec + 32 + PCL_DRAPE_WORDS;
  Drape walls = load_drape(rec + 32);
  Plot plot;                                 // not step_plot(): it reorders this kernel's code
  {
    const int32_t* r = rec + 48;
    plot.frame = r[PCL_P_FRAME]; plot.error = r[PCL_P_ERROR];
    plot.order_r = r[PCL_P_ORDER_R]; plot.order_c = r[PCL_P_ORDER_C];
    plot.order_frame = r[PCL_P_ORDER_FRAME]; plot.ego_mask = r[PCL_P_EGO_MASK];
  }

  const ScrollyCfg wcfg = scrolly_cfg(H, W, p.PH, p.PW, p.margin[0][0], p.margin[0][1]);
  const ScrollyCfg ccfg = scrolly_cfg(H, W, p.PH, p.PW, p.margin[1][0], p.margin[1][1]);
  Directives dir = fresh_directives();
  const int motion = action_to_motion(action);

  plot.frame += 1;                                           // engine.py:716

  // ---- 2. update group 0: '#' MazeDrape (scrolly_maze.py:308-329) --------
  if (motion != PCL_M_NONE)
    scrolly_move_p(walls, wcfg, motion, plot, p_row, p_col, p_permit, p_permit_frame);
  const bool ordered = plot.order_frame == plot.frame;
  const int wr = walls.corner_r, wc = walls.corner_c;
  // Where the '@' window will be after it obeys the same order (checked below).
  const int cr_pred = rec_coins[PCL_D_CORNER_R] + (ordered && motion != PCL_M_NONE ? plot.order_r : 0);
  const int cc_pred = rec_coins[PCL_D_CORNER_C] + (ordered && motion != PCL_M_NONE ? plot.order_c : 0);

  // ---- 3. one batch of loads ---------------------------------------------
  const int we = (wc >> 5) & ~1, ce = (cc_pred >> 5) & ~1;   // first staged word (even)
  const bool narrow = narrow_board(pitch);   // the 4-word fast paths
  // '@' has not moved yet this frame: its pre-scroll corner as scrolly_touch_prescroll
  // will leave it in group 2.
  const bool c_touch = rec_coins[PCL_D_LAST_FRAME] < plot.frame;
  const int c_pre_r = rec_coins[c_touch ? PCL_D_CORNER_R : PCL_D_PRE_R];
  const int c_pre_c = rec_coins[c_touch ? PCL_D_CORNER_C : PCL_D_PRE_C];
  // Delta rendering: neither window moves and the board is this env's last render.
  bool delta = key_ok && !restart && wr == rec[32 + PCL_D_CORNER_R] &&
               wc == rec[32 + PCL_D_CORNER_C] && cr_pred == rec_coins[PCL_D_CORNER_R] &&
               cc_pred == rec_coins[PCL_D_CORNER_C] && rec_coins[PCL_D_AUX2] != -1;
  // The patch trip: one job and at most two words per lane.  Every lane computes its
  // address, predicates, shift and mask with selects, issues both loads, and only then
  // combines them, so the step waits on one round trip here, not one per kind of job.
  //   lanes 0..3    walker `lane`'s 5x5 wall word (see "Wall neighbourhoods"): covers
  //                 every cell any _check_motion of this step can consult, wherever the
  //                 scroll order moves the walker first;
  //   lanes 4..6    row lane - 4 of the 3x3 coin patch around the player at the pre-scroll
  //                 corner, lane 7 the coin bit at that corner (an off-board player sits
  //                 at (0, 0));
  //   lanes 8..19   delta only: 3 coin bits of row k around sprite s's start cell
  //                 (lane 8 + 3 s + k);
  //   lanes 20..31  delta only: 3 backdrop bytes of row k around sprite s's start cell
  //                 (lane 20 + 3 s + k), from the two aligned words that hold them.
  // A clean group's coin row comes from the level's template (see "Coin groups").
  uint32_t got;
  {
    const bool wall_lane = lane < 4, coin_lane = lane < 20, pc_lane = lane < 8;
    const int j = coin_lane ? lane - 8 : lane - 20;          // delta jobs: 3 s + k
    const int s = wall_lane ? lane : pc_lane ? 0 : j / 3;
    const int vr = rec[s * PCL_SPRITE_WORDS + PCL_S_VROW], vc = rec[s * PCL_SPRITE_WORDS + PCL_S_VCOL];
    // board row of a coin or backdrop job, and the first column it reads
    const int r = pc_lane ? (lane < 7 ? p_vrow + lane - 5 : 0) : vr + j - 3 * (j / 3) - 1;
    const int c = pc_lane ? (lane < 7 ? c_pre_c + p_vcol - 1 : c_pre_c)
                          : coin_lane ? cc_pred + vc - 1 : vc - 1;
    const bool row_ok = (unsigned)r < (unsigned)H && (pc_lane || delta);
    // coin jobs
    const int pr = (pc_lane ? c_pre_r : cr_pred) + r;
    const uint32_t* coin_row =
        (((unsigned)rec_coins[PCL_D_AUX2] >> (pr >> coin_group_shift(p.PH))) & 1u
             ? env_coins(p, env) : level_coins(p, lvl)) + (int64_t)pr * PWW;
    // wall jobs: the centre (pattern row, column) of the walker's patch
    const int wr_c = wr + vr + 2, wc_c = wc + vc + 2;       // + the table's 2-cell margin
    const int tw = p.PW + 4;
    const uint32_t* base =
        wall_lane ? p.derived[2] + lvl * p.derived_bstride[2] + (int64_t)wr_c * tw + wc_c
        : coin_lane ? coin_row
                    : reinterpret_cast<const uint32_t*>(p.st.d_backdrop + lvl * p.st.backdrop_bstride +
                                                        (int64_t)r * pitch);
    const int words = coin_lane ? PWW : pitch >> 2;          // words in a coin or backdrop row
    const int wi = wall_lane ? 0 : coin_lane ? c >> 5 : c >> 2;   // floor, may be -1
    const bool ok0 = wall_lane ? (unsigned)wr_c < (unsigned)(p.PH + 4) && (unsigned)wc_c < (unsigned)tw
                               : row_ok && (unsigned)wi < (unsigned)words;
    const bool ok1 = !wall_lane && row_ok && (unsigned)(wi + 1) < (unsigned)words;
    const int sh = wall_lane ? 0 : coin_lane ? c & 31 : (c & 3) * 8;
    // coin bits are not masked to the board here (coin9 is, below; delta candidates off
    // the board fall back); backdrop bytes off the board read 0
    uint32_t mask = wall_lane ? ~0u : lane == 7 ? 1u : 7u;
    if (!coin_lane) {
      mask = 0;
#pragma unroll
      for (int i = 0; i < 3; ++i) mask |= ((unsigned)(c + i) < (unsigned)W ? 0xffu : 0u) << (8 * i);
    }
    const uint64_t keep = l2_evict_last();
    const uint32_t lo = ok0 ? ld_keep(base + wi, keep) : 0u;
    const uint32_t hi = ok1 ? ld_keep(base + wi + 1, keep) : 0u;
    got = __funnelshift_r(lo, hi, sh) & mask;
  }
  const unsigned field = __shfl_sync(PCL_FULL, got, me);   // my walker's 5x5, bit (dr+2)*5 + dc+2
  unsigned coin9 = 0;                        // 3x3 around the player's start + the (0,0) cell
  {
    unsigned colmask = 0;
#pragma unroll
    for (int i = 0; i < 3; ++i)
      colmask |= ((unsigned)(p_vcol - 1 + i) < (unsigned)W ? 1u : 0u) << i;
#pragma unroll
    for (int k = 0; k < 3; ++k) coin9 |= (__shfl_sync(PCL_FULL, got, 4 + k) & colmask) << (3 * k);
    coin9 |= __shfl_sync(PCL_FULL, got, 7) << 9;
  }
  PCL_STAMP(kStPatch);
  uint32_t* s_nb = reinterpret_cast<uint32_t*>(s_bd);   // delta rendering's scratch
  // The bulk copies: the backdrop tile and the two windows -> smem, no registers held.
  // They are first needed after group 2, so they are issued only now: issued ahead of
  // the record and patch loads (as before), every warp's 6 KB of copies queued in front of
  // those two dependent round trips, and in a full wave each trip took 2-4x as long as
  // in a lone warp (tools/step_phases.py; DESIGN.md section 5).  Delta rendering stages
  // nothing unless it falls back to the full paint after group 2.  The paint loop's selector
  // table travels with these copies: the delta path never reads it, and copied at entry
  // by every warp of a wave it was 2 MB per 4096-env launch, all from the same 512 bytes.
  auto stage = [&](int64_t lvl) {
    cp_async16_l1(reinterpret_cast<uint8_t*>(s_sel) + lane * 16,
                  reinterpret_cast<const uint8_t*>(g_sel.v) + lane * 16);
    {
      const uint8_t* src = p.st.d_backdrop + lvl * p.st.backdrop_bstride + lane * 16;
      uint8_t* dst = s_bd + lane * 16;
      const int n16 = (H * pitch) >> 4;
#pragma unroll 4
      for (int i = lane; i < n16; i += 32, src += 512, dst += 512) cp_async16(dst, src);
    }
    // Both windows come from the row-blocked copies (see "Row-blocked windows"): the H rows
    // of a window are one contiguous run there.  Coin window rows of clean groups come from
    // the level's template (see "Coin groups"): per env that is L2 traffic shared by the
    // level's envs instead of DRAM of its own.
    {
      const int gs = coin_group_shift(p.PH);
      const uint32_t* wsrc =
          p.derived[0] + lvl * p.derived_bstride[0] + ((int64_t)(we >> 1) * p.PH + wr) * nw;
      const uint32_t* csrc =
          p.derived[1] + lvl * p.derived_bstride[1] + ((int64_t)(ce >> 1) * p.PH + cr_pred) * nw;
      const int hw = nw >> 1, nhalf = H * hw;  // 8-byte halves per window row
      if (narrow) {                            // one 16-byte row per copy
#pragma unroll 1
        for (int r = lane; r < H; r += 32) {
          cp_async16(s_wall + r * 4, wsrc + r * 4);
          if (!(((unsigned)rec_coins[PCL_D_AUX2] >> ((cr_pred + r) >> gs)) & 1u))
            cp_async16(s_coin + r * 4, csrc + r * 4);
        }
      } else {
#pragma unroll 1
        for (int i = lane; i < nhalf; i += 32) {
          const int pr = cr_pred + i / hw;
          cp_async8(s_wall + i * 2, wsrc + i * 2);
          if (!(((unsigned)rec_coins[PCL_D_AUX2] >> (pr >> gs)) & 1u))
            cp_async8(s_coin + i * 2, csrc + i * 2);
        }
      }
      if (rec_coins[PCL_D_AUX2] != 0) {
#pragma unroll 1
        for (int i = lane; i < nhalf; i += 32) {
          const int r = narrow ? i >> 1 : i / hw, k = (i - r * hw) * 2, pr = cr_pred + r;
          if (((unsigned)rec_coins[PCL_D_AUX2] >> (pr >> gs)) & 1u)
            cp_async8(s_coin + i * 2, env_coins(p, env) + (int64_t)pr * PWW + ce + k);
        }
      }
    }
  };
  if (delta) {
    if (lane < 4) s_nb[kNbWall + lane] = got;
    if (lane >= 8) s_nb[kNbCoin + lane - 8] = got;   // coin rows, then backdrop rows
    if (lane < 4) {
      uint32_t* q = s_nb + kNbStart + 4 * lane;
      q[0] = mine.vrow; q[1] = mine.vcol;
      q[2] = visible(mine) ? mine.row : -1; q[3] = mine.col;
    }
    if (lane < 2) s_nb[kNbStale + lane] = rec_coins[PCL_D_AUX0 + lane];
  } else {
    stage(lvl);
    PCL_STAMP_PATH(restart ? kPathRestart : kPathFull);
  }

  // ---- 4a. update group 1: patrollers a, b, c then P, ONE WALKER PER LANE ----
  // The four walkers do not interact within a frame: each reads the board of
  // render #1 (walls at the new corner, P painted where the previous render put it)
  // and the shared plot; P moves last, so patrollers compare with its OLD virtual
  // position.  (sprites.py:356-477, scrolly_maze.py:258-305.)
  const int r0 = mine.vrow, c0 = mine.vcol;
  const bool is_p = me == 0;
  const bool even = (plot.frame % 2) == 0;
  if (even) scrolly_touch_prescroll(walls, plot);           // PatrollerSprite :291
  int my_err = 0;
  bool hit = false;
  int mot;                                   // this lane's motion this frame
  if (is_p) {
    mot = motion;                            // PCL_M_NONE: P does not move at all (:258)
  } else if (!even) {
    mot = PCL_M_STAY;
  } else {
    const int step = mine.aux0 ? 1 : -1;
    int pr = r0 + walls.pre_r, pc = c0 + walls.pre_c + step;
    bool next_to_wall = false;
    if ((unsigned)pr < (unsigned)p.PH && (unsigned)pc < (unsigned)p.PW) {
      // Same cell seen from the post-scroll corner: inside the 5x5 patch.
      const int dr = pr - wr - r0 + 2, dc = pc - wc - c0 + 2;
      next_to_wall = (field >> (dr * 5 + dc)) & 1u;
    } else {
      // NumPy indexing: negatives wrap once, anything else is an IndexError.
      if (pr < 0) pr += p.PH;
      if (pc < 0) pc += p.PW;
      if ((unsigned)pr < (unsigned)p.PH && (unsigned)pc < (unsigned)p.PW)
        next_to_wall = bit_at(level_walls(p, level_of(p, env)) + (int64_t)pr * PWW, pc);
      else
        my_err |= PCL_ENV_ERR_INDEX;
    }
    if (next_to_wall) mine.aux0 = !mine.aux0;
    mot = mine.aux0 ? PCL_M_E : PCL_M_W;
  }
  if (mot != PCL_M_NONE) {                   // sprites.py:356-389 `_move`
    const int dr = motion_dr(mot), dc = motion_dc(mot);
    if (ordered) {                           // _obey_scrolling_order :413-454
      walker_teleport(mine, H, W, mine.vrow - plot.order_r, mine.vcol - plot.order_c);
      if (is_p && plot.order_r != dr && plot.order_c != dc) my_err |= PCL_ENV_ERR_ORDER_MISMATCH;
    }
    bool legal = true;
    unsigned blk = 0;
    if (mot != PCL_M_STAY || is_p) {
      blk = blocked3x3(mine.vrow, mine.vcol, r0, c0, field, H, W, p_vis, p_row, p_col);
      legal = motion_legal(blk, mot);
    }
    if (legal && mot != PCL_M_STAY) {
      walker_teleport(mine, H, W, mine.vrow + dr, mine.vcol + dc);      // _raw_move :391
      if (is_p) blk = blocked3x3(mine.vrow, mine.vcol, r0, c0, field, H, W, p_vis, p_row, p_col);
    }
    if (is_p) {                              // :456-477 + scrolling.py:373-434
      const int valid_at = plot.frame + 1;
      if (mine.aux1 != valid_at) { mine.aux1 = valid_at; mine.aux0 = 0; }
      mine.aux0 |= legal_motions(blk);
    } else if (even) {
      hit = mine.vrow == p_vrow && mine.vcol == p_vcol;     // PatrollerSprite :303-305
    }
  }
  __syncwarp();                              // every lane has read the records it needs (racecheck)
  if (lane < 4)                              // write my walker back
    store_sprite(rec + me * PCL_SPRITE_WORDS, mine, is_p ? PCL_S_AUX2 : PCL_S_AUX1);
  if (motion != PCL_M_NONE) plot.ego_mask |= 1;             // sprites.py:443 (P only)
  plot.error |= __reduce_or_sync(PCL_FULL, (unsigned)(lane < 4 ? my_err : 0));
  if (__any_sync(PCL_FULL, lane < 4 && hit)) terminate(dir);
  // The player after its move, for everything below.
  Sprite pl;
  pl.row = __shfl_sync(PCL_FULL, mine.row, 0); pl.col = __shfl_sync(PCL_FULL, mine.col, 0);
  pl.vrow = __shfl_sync(PCL_FULL, mine.vrow, 0); pl.vcol = __shfl_sync(PCL_FULL, mine.vcol, 0);
  pl.flags = __shfl_sync(PCL_FULL, mine.flags, 0);
  pl.aux0 = __shfl_sync(PCL_FULL, mine.aux0, 0); pl.aux1 = __shfl_sync(PCL_FULL, mine.aux1, 0);

  // ---- 4b. update group 2: '@' CashDrape (scrolly_maze.py:341-364) -------
  Drape coins = load_drape(rec_coins);
  scrolly_touch_prescroll(coins, plot);
  plot.aux0 = rec[48 + PCL_P_AUX0];
  int picked_r = -1, picked_c = -1;          // pattern cell cleared this frame
  {
    const int dr = pl.row - p_vrow, dc = pl.col - p_vcol;
    bool coin;
    const int pr = coins.pre_r + pl.row, pc = coins.pre_c + pl.col;
    if (pl.row == 0 && pl.col == 0 && !on_board(pl.vrow, pl.vcol, H, W))
      coin = (coin9 >> 9) & 1u;              // off-board player sits at (0, 0)
    else if ((unsigned)(dr + 1) <= 2u && (unsigned)(dc + 1) <= 2u)
      coin = (coin9 >> ((dr + 1) * 3 + dc + 1)) & 1u;
    else
      coin = bit_at(env_coins(p, env) + (int64_t)pr * PWW, pc);   // cannot happen
    if (coin) {
      add_reward(dir, 100);
      // A reduction with no result (RED): nothing on this warp waits for the word's old
      // value, where a read-modify-write put one more round trip on the pick-up's step.
      if (lane == 0) atomicAnd(env_coins(p, env) + (int64_t)pr * PWW + (pc >> 5), ~(1u << (pc & 31)));
      picked_r = pr; picked_c = pc;
      plot.aux0 -= 1;
      if (plot.aux0 == 0) terminate(dir);
      coins.aux0 = pl.row; coins.aux1 = pl.col;         // stale until next refresh
    }
  }
  if (motion != PCL_M_NONE) {
    scrolly_move_p(coins, ccfg, motion, plot, pl.row, pl.col, pl.aux0, pl.aux1);
    coins.aux0 = -1; coins.aux1 = -1;                    // _update_curtain :689
  } else if (action == 5) {
    terminate(dir);
  }
  PCL_STAMP(kStGroup2);

  // ---- _apply_and_clear_plot (engine.py:761-847); no z-order changes here.
  cp_async_wait_all();
  PCL_STAMP(kStWait);
  __syncwarp();
  if (lane == 0) {
    // The env's episode return so far (store_episode below), in this lane only and behind
    // the pointer test, so that with nothing bound the step's path is the one without it.
    const double ep_so_far = load_episode(p, env);
    store_drape(rec + 32, walls, PCL_D_AUX0);
    store_drape(rec + 32 + PCL_DRAPE_WORDS, coins, PCL_D_AUX2);
    apply_time_limit(p, plot, dir);
    store_episode(p, env, plot.frame, ep_so_far, (double)dir.reward);
    store_plot<ORDER_ALL>(rec + 48, plot, dir);
    rec[48 + PCL_P_AUX0] = plot.aux0;
    store_outputs(p.out, env, dir);
    // The pick-up's group of the env's pattern now differs from the template.
    if (picked_r >= 0) rec[32 + PCL_DRAPE_WORDS + PCL_D_AUX2] |= 1 << (picked_r >> coin_group_shift(p.PH));
  }
  const int cr = coins.corner_r, cc = coins.corner_c;

  // ---- 4c. delta rendering: store the final value of every cell that can have changed.
  // Candidates, one per lane: the old (lanes 0..3) and new (4..7) cells of the sprites,
  // the old (8) and new (9) stale coin, and the coin picked up (10).  With both windows
  // where they were, every other cell shows the walls, coins, backdrop and sprites it
  // showed in the last render.  A cell listed twice gets the same value twice.  A moved
  // '@' window or a candidate outside the loaded neighbourhoods falls back to the full
  // paint, staged only now.
  if (delta) {
    __syncwarp();                            // the new records are in rec
    bool fall = cr != cr_pred || cc != cc_pred;
    int cell = -1;
    uint32_t val = 0;
    if (!fall) {
      int r = -1, c = -1;
      if (lane < 4) {
        r = (int)s_nb[kNbStart + 4 * lane + 2]; c = (int)s_nb[kNbStart + 4 * lane + 3];
      } else if (lane < 8) {
        const int32_t* s = rec + (lane - 4) * PCL_SPRITE_WORDS;
        if (s[PCL_S_FLAGS] & 1) { r = s[PCL_S_ROW]; c = s[PCL_S_COL]; }
      } else if (lane == 8) {
        r = (int)s_nb[kNbStale]; c = (int)s_nb[kNbStale + 1];
      } else if (lane == 9) {
        r = rec_coins[PCL_D_AUX0]; c = rec_coins[PCL_D_AUX1];
      } else if (lane == 10 && picked_r >= 0) {
        r = picked_r - cr; c = picked_c - cc;
      }
      bool outside = false;
      if (r >= 0) {
        int s = -1, dr = 0, dc = 0;          // a sprite whose 3x3 holds (r, c), at (dr, dc)
#pragma unroll
        for (int t = kS - 1; t >= 0; --t) {
          const int a = r - (int)s_nb[kNbStart + 4 * t] + 1, b = c - (int)s_nb[kNbStart + 4 * t + 1] + 1;
          if ((unsigned)a <= 2u && (unsigned)b <= 2u) { s = t; dr = a; dc = b; }
        }
        outside = s < 0 || !on_board(r, c, H, W);
        if (!outside) {
          // z-order a b c @ # P, as the full paint composes it
          const bool wall = (s_nb[kNbWall + s] >> ((dr + 1) * 5 + dc + 1)) & 1u;
          bool coin = (s_nb[kNbCoin + 3 * s + dr] >> dc) & 1u;
          if (picked_r - cr == r && picked_c - cc == c) coin = false;
          if (rec_coins[PCL_D_AUX0] == r && rec_coins[PCL_D_AUX1] == c) coin = true;
          val = (s_nb[kNbBackdrop + 3 * s + dr] >> (8 * dc)) & 0xffu;
          // t = 1..3: a, b, c; t = 4: '@', '#', then P (sprite 0) on top
#pragma unroll
          for (int t = 1; t <= kS; ++t) {
            const int32_t* q = rec + (t & 3) * PCL_SPRITE_WORDS;
            if (t == kS && coin) val = '@';
            if (t == kS && wall) val = '#';
            if ((q[PCL_S_FLAGS] & 1) && q[PCL_S_ROW] == r && q[PCL_S_COL] == c) val = p.sprite_char[t & 3];
          }
          cell = r * pitch + c;
        }
      }
      fall = __any_sync(PCL_FULL, outside);
    }
    if (fall) {
      __syncwarp();                          // every lane is done with the scratch words
      delta = false;
      stage(level_of(p, env));
      cp_async_wait_all();
      PCL_STAMP_PATH(kPathFellBack);
    } else if (cell >= 0) {
      p.out.d_board[(int64_t)env * H * pitch + cell] = (uint8_t)val;
    }
  }

  // The coin window was staged before the pick-up: clear the bit there too.
  if (!delta && lane == 0 && picked_r >= 0) {
    const int r2 = picked_r - cr_pred, b = picked_c - (ce << 5);
    if ((unsigned)r2 < (unsigned)H && (unsigned)b < (unsigned)(nw * 32))
      s_coin[r2 * nw + (b >> 5)] &= ~(1u << (b & 31));
  }
  int ce_final = ce;
  if (cr != cr_pred || cc != cc_pred) {      // '@' issued its own order: restage
    __syncwarp();
    ce_final = (cc >> 5) & ~1;
    for (int i = lane; i < H * nw; i += 32)
      s_coin[i] = env_coins(p, env)[(int64_t)(cr + i / nw) * PWW + ce_final + i % nw];
  }
  __syncwarp();
  p.st.d_sprites[(int64_t)env * kS * PCL_SPRITE_WORDS + lane] = rec[lane];
  if (lane < 16) p.st.d_drapes[(int64_t)env * 2 * PCL_DRAPE_WORDS + lane] = rec[32 + lane];
  else p.st.d_plot[(int64_t)env * PCL_PLOT_WORDS + lane - 16] = rec[32 + lane];
  if (lane < kKeyWords)                      // what the board in d_board is now drawn from
    p.render_key[(int64_t)env * kKeyStride + lane] = key_word(rec, lane, p.board_epoch, pitch);
  if (delta) {                               // 4c stored every cell that changed
    PCL_STAMP_PATH(picked_r >= 0 ? kPathDeltaPickup : kPathDelta);
    PCL_STAMP(kStPatched);
    PCL_STAMP(kStPaint);
    if (p.has_cropper) {
      __syncwarp();
      crop_epilogue(p.cropper, p.out.d_board, env, lane, rec, rec + 48);
    }
    PCL_STAMP(kStEnd);
    PCL_STAMP_TIME(kStTimeOut);
    return;
  }

  // ---- 5. final render, z-order a b c @ # P (engine.py:737-759) ----------
  // 5a. Window rows -> ONE word per 16-cell board segment (wall16 << 16 | coin16),
  // aligned to the board: each lane shifts whole rows once, so the streaming loop
  // below does no bit addressing at all.  Cells past W and the stale coin
  // (drapes.py:689 has not refreshed the curtain yet) are folded in here.
  const int spr = pitch >> 4;                // 16-byte segments per row
  // Narrow boards keep the segment words where the wall window rows were.
  uint32_t* s_seg = narrow ? s_wall : s_coin + ((H * nw + 3) & ~3);
  const int wsh = wc - (we << 5), csh = cc - (ce_final << 5);     // 0..63 into the staged row
  if (narrow) {
    const uint32_t m_lo = W >= 32 ? 0xffffffffu : (1u << W) - 1u;
    const uint32_t m_hi = W >= 64 ? 0xffffffffu : W > 32 ? (1u << (W - 32)) - 1u : 0u;
    // Row r's segment words land in the wall slot of row spr * r / 4 <= r, which may be
    // another lane's row of the same round: every lane reads its rows before any lane
    // stores.  A round stores nothing past its own rows, so later rounds read intact slots.
    for (int r0 = 0; r0 < H; r0 += 32) {
      const int r = min(r0 + lane, H - 1);   // lanes past the last row redo it, store nothing
      const uint4 wv = *reinterpret_cast<const uint4*>(s_wall + r * 4);
      const uint4 cv = *reinterpret_cast<const uint4*>(s_coin + r * 4);
      const uint32_t wa = (wsh & 32) ? wv.y : wv.x, wb = (wsh & 32) ? wv.z : wv.y,
                     wd = (wsh & 32) ? wv.w : wv.z;
      const uint32_t ca = (csh & 32) ? cv.y : cv.x, cb = (csh & 32) ? cv.z : cv.y,
                     cd = (csh & 32) ? cv.w : cv.z;
      const uint32_t w_lo = __funnelshift_r(wa, wb, wsh & 31) & m_lo;
      const uint32_t w_hi = __funnelshift_r(wb, wd, wsh & 31) & m_hi;
      const uint32_t c_lo = __funnelshift_r(ca, cb, csh & 31) & m_lo;
      const uint32_t c_hi = __funnelshift_r(cb, cd, csh & 31) & m_hi;
      __syncwarp();
      if (r0 + lane < H) {
        uint32_t* out = s_seg + r * spr;
        out[0] = __byte_perm(c_lo, w_lo, 0x5410);
        if (spr > 1) out[1] = __byte_perm(c_lo, w_lo, 0x7632);
        if (spr > 2) out[2] = __byte_perm(c_hi, w_hi, 0x5410);
        if (spr > 3) out[3] = __byte_perm(c_hi, w_hi, 0x7632);
      }
    }
  } else {                                   // general width: one (row, segment) per lane and round
    for (int i = lane; i < H * spr; i += 32) {
      const int r = i / spr, j = i - r * spr;
      const int ncols = min(16, W - 16 * j);
      if (ncols <= 0) { s_seg[i] = 0; continue; }          // pitch padding past the board
      const uint32_t keep = (1u << ncols) - 1u;
      const int wo = wsh + 16 * j, co = csh + 16 * j;
      const uint32_t* wrow = s_wall + r * nw;
      const uint32_t* crow = s_coin + r * nw;
      // the second word is only fetched while inside the staged row
      const uint32_t w16 = __funnelshift_r(wrow[wo >> 5], (wo >> 5) + 1 < nw ? wrow[(wo >> 5) + 1] : 0u,
                                           wo & 31) & keep;
      const uint32_t c16 = __funnelshift_r(crow[co >> 5], (co >> 5) + 1 < nw ? crow[(co >> 5) + 1] : 0u,
                                           co & 31) & keep;
      s_seg[i] = (w16 << 16) | c16;
    }
  }
  // a, b, c lie under both drapes, so they are patched into the staged backdrop
  // up front, in z-order (a lane each, one after the other); the player is the TOP
  // layer: its character also goes into the staged tile, and both drape bits of its
  // cell are cleared so that the compose below keeps the tile's byte there — the
  // streaming loop then has no sprite test at all.
  __syncwarp();
  if (lane == 0 && coins.aux0 >= 0)
    s_seg[coins.aux0 * spr + (coins.aux1 >> 4)] |= 1u << (coins.aux1 & 15);
#pragma unroll
  for (int i = 1; i < kS; ++i) {
    if (lane == i && visible(mine)) s_bd[mine.row * pitch + mine.col] = p.sprite_char[i];
    __syncwarp();
  }
  if (lane == 0 && visible(pl)) {
    s_bd[pl.row * pitch + pl.col] = p.sprite_char[0];
    s_seg[pl.row * spr + (pl.col >> 4)] &= ~(0x00010001u << (pl.col & 15));
  }
  __syncwarp();                              // (also: this warp's s_sel copy has landed, waited above)
  PCL_STAMP(kStPatched);
  // 5b. The streaming loop: 16 cells per lane per iteration, segment index ==
  // 16-byte index into both the staged tile and the board (pitch = 16 * spr).
  const int total = H * spr;
  const unsigned drape_chars = ('#' << 8) | '@';           // bytes 4 and 5 of the permute
  const uint4* src = reinterpret_cast<const uint4*>(s_bd);
  uint4* dst = reinterpret_cast<uint4*>(p.out.d_board + (int64_t)env * H * pitch);
  for (int seg = lane; seg < total; seg += 32) {
    uint4 px = src[seg];
    const uint32_t bits = s_seg[seg];
    px.x = prmt(px.x, drape_chars, s_sel[((bits >> 12) & 0xf0u) | (bits & 0xfu)]);
    px.y = prmt(px.y, drape_chars, s_sel[((bits >> 16) & 0xf0u) | ((bits >> 4) & 0xfu)]);
    px.z = prmt(px.z, drape_chars, s_sel[((bits >> 20) & 0xf0u) | ((bits >> 8) & 0xfu)]);
    px.w = prmt(px.w, drape_chars, s_sel[((bits >> 24) & 0xf0u) | ((bits >> 12) & 0xfu)]);
    dst[seg] = px;
  }
  PCL_STAMP(kStPaint);
  // ---- 6. an attached cropper (pcl_attach_cropper): the egocentric view of the board
  // this warp has just stored, without a second kernel (ScrollingCropper.crop,
  // cropping.py:393-426).
  if (p.has_cropper) {
    __syncwarp();
    crop_epilogue(p.cropper, p.out.d_board, env, lane, rec, rec + 48);
  }
  PCL_STAMP(kStEnd);
  PCL_STAMP_TIME(kStTimeOut);
}

__global__ void __launch_bounds__(kWarpsPerBlock * 32, 8)
scrolly_maze_step(const StepParams p) {
  PCL_STAMP(kStEntry);
  PCL_STAMP_TIME(kStTimeIn);
  // Entry of "Block chaining": nothing before it reads state earlier kernels may produce.
  // begin[b], end[b] at block_sync[2 b], [2 b + 1]
  __shared__ uint32_t s_begun;
  if (p.chain == CHAIN_NONE) {
    pdl_launch_dependents();
    pdl_wait_prior_grids();
    PCL_STAMP(kStPrior);
    step_env(p);
    return;
  }
  uint32_t* const sync = p.block_sync + 2 * blockIdx.x;
  if (threadIdx.x == 0) s_begun = atomicAdd(sync, 1u);
  if (p.chain == CHAIN_HEAD) {
    pdl_wait_prior_grids();
  } else if (threadIdx.x == 0) {
    while (ld_relaxed_gpu(sync + 1) != s_begun) __nanosleep(64);
    ld_acquire_gpu(sync + 1);              // reads that same count: what those blocks wrote
  }
  __syncthreads();
  pdl_launch_dependents();
  PCL_STAMP(kStPrior);
  step_env(p);
  __syncthreads();
  // end[b] == begun before this launch (the full wait, or the spin): now one more.
  if (threadIdx.x == 0) st_release_gpu(p.block_sync + 2 * blockIdx.x + 1, s_begun + 1u);
}

// Dynamic shared memory of one block (kWarpsPerBlock envs).
size_t block_smem(int H, int W, int pitch) {
  return warp_smem_bytes(H, W, pitch) * kWarpsPerBlock;
}

int check_spec(const pcl_spec& s) {
  if (!chars_are(s.sprite_char, s.n_sprites, "Pabc")) return PCL_ERR_UNSUPPORTED;
  if (!chars_are(s.drape_char, s.n_drapes, "#@")) return PCL_ERR_UNSUPPORTED;
  if (!chars_are(s.z_order, 6, "abc@#P")) return PCL_ERR_UNSUPPORTED;
  const int lens[3] = {1, 4, 1};
  if (!groups_are(s, "#abcP@", lens, 3)) return PCL_ERR_UNSUPPORTED;
  for (int i = 0; i < 4; ++i) {
    if (!set_is(s.impassable[i], "#")) return PCL_ERR_UNSUPPORTED;
    if (s.sprite_confined[i]) return PCL_ERR_UNSUPPORTED;
    if (s.sprite_egocentric[i] != (i == 0)) return PCL_ERR_UNSUPPORTED;
  }
  if (s.pattern_rows < s.rows || s.pattern_cols < s.cols) return PCL_ERR_INVALID;
  {
    // Window rows are staged from the even word at or below corner_c >> 5:
    // window_words(W) words (4 up to 64 columns) must stay inside the row.
    const int nw = window_words(s.cols);
    if ((s.pattern_words & 1) || s.pattern_words < (((s.pattern_cols - s.cols) >> 5) & ~1) + nw ||
        s.pattern_words < (s.pattern_cols + 31) / 32 + 1) return PCL_ERR_INVALID;
    // one CTA (4 envs) stages tile + windows in shared memory: the launcher's own size
    if (block_smem(s.rows, s.cols, s.pitch) > kMaxDynamicSmem) return PCL_ERR_UNSUPPORTED;
  }
  for (int d = 0; d < 2; ++d)
    if (!margins_fit(s, d)) return PCL_ERR_INVALID;
  return PCL_OK;
}

int check_state(const pcl_spec&, const pcl_state& st) {
  for (int d = 0; d < 2; ++d) if (!st.d_pattern[d]) return PCL_ERR_INVALID;
  if (!st.d_pattern_init[1] || st.pattern_bstride[1] == 0) return PCL_ERR_INVALID;
  return PCL_OK;
}

// '#' is a window of its pattern; '@' too, less the coin its record names as stale.
CurtainAt curtain(const pcl_spec&, int d) {
  return d == 1 ? CurtainAt::kStaleWindow : CurtainAt::kPatternWindow;
}

cudaError_t launch(const StepParams& p, cudaStream_t s) {
  if (p.PWW & 1) return cudaErrorInvalidValue;   // window rows are staged in 8-byte halves
  const size_t smem = block_smem(p.H, p.W, p.pitch);
  if (smem > kMaxDynamicSmem) return cudaErrorInvalidValue;   // board too large for one CTA
  // Programmatic dependent launch: this kernel may start (prologue only) before
  // the previous kernel of the stream has drained.
  return launch_step(scrolly_maze_step, p, kWarpsPerBlock, smem, s, /*pdl=*/true);
}

// ---- Row-blocked windows (built by derive() for each pcl_bind_state) -----------------
// Block k of a pattern holds words [2k, 2k + window_words(W)) of every pattern row, rows
// contiguous, so the window at first word 2k and row r0 is ONE run of H * window_words(W)
// words.  Staged from the pattern itself, a 16-byte window row fills only half of the
// 32-byte L2 sector it is read from whenever pattern rows are 32 bytes or more apart.
// Blocks exist for every first word a window can stage, 0 .. ((PW - W) >> 5) & ~1.  One
// copy of the wall pattern d_pattern[0] (derived[0]) and one of the coin template
// d_pattern_init[1] (derived[1]), each indexed like the array it comes from.

__global__ void build_blocked(const uint32_t* src, int64_t src_bstride, uint32_t* dst, int PH,
                              int PWW, int nw, int nblk, int64_t total) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    int64_t t = i / nw;
    const int w = (int)(i - t * nw);
    const int row = (int)(t % PH);
    t /= PH;
    const int k = (int)(t % nblk);
    dst[i] = src[(t / nblk) * src_bstride + (int64_t)row * PWW + 2 * k + w];
  }
}

// ---- Wall neighbourhoods (built by derive() beside the row-blocked windows) ----------
// One word per pattern cell (pr, pc), with a 2-cell margin: word (pr + 2) * (PW + 4) +
// pc + 2 of a copy has bit (dr + 2) * 5 + dc + 2 set iff the wall pattern has a wall at
// (pr + dr, pc + dc), where rows outside [0, PH), negative columns and columns past the
// row's PWW words read 0 (columns in [PW, 32 PWW) read the row's zero padding).  So a
// walker's whole 5x5 patch is one load.  A centre outside the margin reads 0 in all 25
// cells: the kernel loads nothing for it.  (PH + 4) * (PW + 4) words per copy, one per
// level (one per env without a level index), or a single one when the pattern has no
// stride: derived[2].
__global__ void build_neighbourhoods(const uint32_t* src, int64_t src_bstride, uint32_t* dst, int PH,
                                     int PW, int PWW, int64_t total) {
  const int tw = PW + 4;
  const int64_t per_copy = (int64_t)(PH + 4) * tw;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t t = i / per_copy;
    const int cell = (int)(i - t * per_copy);
    const int pr = cell / tw - 2, c_first = cell % tw - 4;   // first column of each patch row
    const int wi = c_first >> 5;                             // floor, may be -1
    uint32_t word = 0;
    for (int k = 0; k < 5; ++k) {
      const int r = pr + k - 2;
      if ((unsigned)r >= (unsigned)PH) continue;
      const uint32_t* row = src + t * src_bstride + (int64_t)r * PWW;
      const uint32_t lo = (unsigned)wi < (unsigned)PWW ? row[wi] : 0u;
      const uint32_t hi = (unsigned)(wi + 1) < (unsigned)PWW ? row[wi + 1] : 0u;
      word |= (__funnelshift_r(lo, hi, c_first & 31) & 31u) << (5 * k);
    }
    dst[i] = word;
  }
}

int derive(const pcl_spec& s, const pcl_state& st, int batch, StepParams* p, void** owned) {
  // Copies of per-level data: as many as the level index can name (one per env without
  // one), or a single one when the array has no stride.
  int64_t levels = batch;
  if (st.d_level) {
    int32_t* lv = new (std::nothrow) int32_t[batch];
    if (!lv) return PCL_ERR_NOMEM;
    const cudaError_t e = cudaMemcpy(lv, st.d_level, sizeof(int32_t) * batch, cudaMemcpyDeviceToHost);
    levels = 1;
    for (int i = 0; e == cudaSuccess && i < batch; ++i) levels = std::max<int64_t>(levels, lv[i] + 1);
    delete[] lv;
    if (e != cudaSuccess) return PCL_ERR_CUDA;
  }
  const int W = s.cols, PH = s.pattern_rows;
  const int nw = window_words(W), nblk = ((((s.pattern_cols - W) >> 5) & ~1) >> 1) + 1;
  const int64_t blk_words = (int64_t)nblk * PH * nw;              // one blocked copy
  const int64_t n_wall = st.pattern_bstride[0] == 0 ? 1 : levels;
  const int64_t n_coin = st.pattern_init_bstride[1] == 0 ? 1 : levels;
  const int64_t nbh_words = (int64_t)(PH + 4) * (s.pattern_cols + 4);   // one neighbourhood copy
  const int64_t off_coin = (n_wall * blk_words * 4 + 255) & ~(int64_t)255;
  const int64_t off_nbh = (off_coin + n_coin * blk_words * 4 + 255) & ~(int64_t)255;
  const int64_t off_key = (off_nbh + n_wall * nbh_words * 4 + 255) & ~(int64_t)255;
  const int64_t off_sync = (off_key + (int64_t)batch * kKeyStride * 4 + 255) & ~(int64_t)255;
  const int64_t sync_bytes = (int64_t)(batch + kWarpsPerBlock - 1) / kWarpsPerBlock * 2 * 4;
  uint8_t* buf = nullptr;
  if (cudaMalloc(&buf, off_sync + sync_bytes) != cudaSuccess) return PCL_ERR_NOMEM;
  *owned = buf;
  uint32_t* wall = reinterpret_cast<uint32_t*>(buf);
  uint32_t* coin = reinterpret_cast<uint32_t*>(buf + off_coin);
  uint32_t* nbh = reinterpret_cast<uint32_t*>(buf + off_nbh);
  // Render keys of no render (frame -1): the first launch paints every board.
  p->render_key = reinterpret_cast<int32_t*>(buf + off_key);
  if (cudaMemset(p->render_key, 0xff, (size_t)batch * kKeyStride * 4) != cudaSuccess) return PCL_ERR_CUDA;
  // No launch of the new binding has begun or ended (see "Block chaining").
  p->block_sync = reinterpret_cast<uint32_t*>(buf + off_sync);
  if (cudaMemset(p->block_sync, 0, sync_bytes) != cudaSuccess) return PCL_ERR_CUDA;
  build_blocked<<<1024, 256>>>(st.d_pattern[0], st.pattern_bstride[0], wall, PH, s.pattern_words,
                               nw, nblk, n_wall * blk_words);
  build_blocked<<<1024, 256>>>(st.d_pattern_init[1], st.pattern_init_bstride[1], coin, PH,
                               s.pattern_words, nw, nblk, n_coin * blk_words);
  build_neighbourhoods<<<1024, 256>>>(st.d_pattern[0], st.pattern_bstride[0], nbh, PH,
                                      s.pattern_cols, s.pattern_words, n_wall * nbh_words);
  p->derived[0] = wall; p->derived_bstride[0] = n_wall > 1 ? blk_words : 0;
  p->derived[1] = coin; p->derived_bstride[1] = n_coin > 1 ? blk_words : 0;
  p->derived[2] = nbh; p->derived_bstride[2] = n_wall > 1 ? nbh_words : 0;
  return cudaDeviceSynchronize() == cudaSuccess && cudaGetLastError() == cudaSuccess ? PCL_OK
                                                                                     : PCL_ERR_CUDA;
}

}  // namespace

const Program kScrollyMaze = {check_spec, check_state, curtain, launch, nullptr,
                              /*float_reward=*/false, /*crop_epilogue=*/true,
                              /*scroll_groups=*/false, /*check_code=*/nullptr,
                              /*float_reward_arg0=*/false, derive, /*block_chaining=*/true};

}  // namespace pcl

// The wall-neighbourhood table derive() builds (see "Wall neighbourhoods"), for `copies`
// wall patterns of rows x words words, `bstride` words apart, into d_dst ((rows + 4) x
// (cols + 4) words per copy), so that tests can hold the table against its rule.  Not
// part of include/pcl.h.  0, or -3 on a CUDA error.
extern "C" int pcl_scrolly_wall_neighbourhoods(const uint32_t* d_pattern, int64_t bstride, int rows,
                                               int cols, int words, int64_t copies, uint32_t* d_dst) {
  pcl::build_neighbourhoods<<<1024, 256>>>(d_pattern, bstride, d_dst, rows, cols, words,
                                           copies * (rows + 4) * (cols + 4));
  return cudaDeviceSynchronize() == cudaSuccess && cudaGetLastError() == cudaSuccess ? 0 : -3;
}

#ifdef PCL_STEP_STAMPS
// Copies the stamps of the last scrolly_maze_step launch for envs [0, n) to host memory
// (n * 12 u32, in the order of the kSt* slots).  Only the stamp build exports it.
extern "C" int pcl_step_stamps(uint32_t* host, int n) {
  if (n < 0 || n > pcl::kStampEnvs) return -1;
  return cudaMemcpyFromSymbol(host, pcl::g_stamps, sizeof(pcl::g_stamps[0]) * n) == cudaSuccess
             ? 0 : -3;
}
#endif
