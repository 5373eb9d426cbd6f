// compiled.cu — the compiled step program: MazeWalkers (egocentric or not), plain Sprites,
// Scrollys and plain drapes whose update() bodies `pycolab_b200.compiler` translated into
// the bytecode of include/pcl.h (PCL_OP_*).
//
// A plain Sprite (program_arg[3]) sets its own position and visibility (PCL_OP_SETFIELD)
// and may stand anywhere: the render wraps its position as NumPy indexing does, and a
// visible one off the board latches PCL_ENV_ERR_INDEX after its update group's render.
//
// Scrollys scroll with fixture.cu's motion helper (board::scrolly_move_dyn), in the one
// scrolling group whose order words live in the plot record.  A Scrolly's curtain is the
// window of its pattern as of its last motion helper (drapes.py:689-695): read from the
// static pattern at its corner, or, for a Scrolly whose code writes its pattern, kept in
// d_bits and copied from the per-env pattern at each motion helper, so a write shows on
// the board only after the next one, as upstream.
//
// The kernel is fixture.cu's frame — one warp per env, a real board in shared memory,
// rendered after every update group (engine.py:725-735) — with an interpreter where the
// fixture reads precomputed motions: each entity runs its class's code over the records
// in shared memory.  Interpretation is warp-uniform: every lane runs the same
// instruction on the same values, and the operand stack and locals live in shared
// memory.  The lanes split up only for a render, a walker's neighbourhood, a curtain
// fill, a curtain's any() and an MT19937 twist.
//
// Draws (PCL_OP_RANDINT / RANDCMP) continue the env's generator words in d_rng, in global
// memory as marauders.cu and shockwave.cu keep theirs: a draw reads one or two words and
// the position, and every 624th output the warp twists the 624 words together.
//
// Semantics restated from upstream:
//   - update() runs on the its_showtime() frame too, with actions=None (engine.py:581);
//   - another entity's record is read as it is now; a curtain write shows in reads at
//     once and on the board at the next render;
//   - Plot directives apply in call order: rewards sum (plot.py:201-214), the last
//     discount-setting call wins, terminate_episode() does not stop later updates.
#include "pcl_board.cuh"
#include "pcl_mt.cuh"

#include <vector>

namespace pcl {

namespace {

constexpr int kWarpsPerBlock = 2;
using board::Ctx;
using board::WarpState;

// The operand stack and locals, in shared memory, one per warp.  Every lane keeps its
// own copy of each slot (slot i of lane l is word i * 32 + l, so the lanes hit 32
// different banks): a lane only ever reads back what it wrote itself, and nothing
// depends on the warp staying converged between instructions.
struct Vm {
  int32_t stack[PCL_CODE_STACK][32];
  int32_t local[PCL_CODE_LOCALS][32];
};

// One lane's view of a column of Vm slots.
struct LaneSlots {
  int32_t* base;                     // slot 0 of this lane
  __device__ __forceinline__ int32_t& operator[](int i) const { return base[i * 32]; }
};

// Operand words of opcode `op` (PCL_OP_IN and PCL_OP_PICK have their count more).
__host__ __device__ __forceinline__ int op_operands(int op) {
  switch (op) {
    case PCL_OP_RANDCMP: return 4;
    case PCL_OP_FIELD: case PCL_OP_REWARD_F64: case PCL_OP_RANDINT: return 2;
    case PCL_OP_PUSH: case PCL_OP_LOAD: case PCL_OP_STORE: case PCL_OP_JMP: case PCL_OP_JZ:
    case PCL_OP_JNZ: case PCL_OP_IN: case PCL_OP_GETR: case PCL_OP_SETR: case PCL_OP_GETP:
    case PCL_OP_SETP: case PCL_OP_CURTAIN: case PCL_OP_ANY: case PCL_OP_MOVE:
    case PCL_OP_TERMINATE: case PCL_OP_DISCOUNT: case PCL_OP_PICK: case PCL_OP_SCROLL:
    case PCL_OP_PRESCROLL: case PCL_OP_POSTSCROLL: case PCL_OP_PATTERN: case PCL_OP_PATANY:
    case PCL_OP_SETFIELD:
      return 1;
    default: return 0;
  }
}

// Operand words of every opcode, the Backdrop's included (host side: pcl_bind_code).  The
// interpreter counts ROLLBACK's itself, so that compiled_step's dispatch stays as it was.
int code_operands(int op) { return op == PCL_OP_ROLLBACK ? 3 : op_operands(op); }

// Stack effect of each opcode (host side: pcl_bind_code's depth check).
struct OpInfo { int8_t pops, pushes; };
constexpr OpInfo kOps[PCL_OP_COUNT] = {
    {0, 0},  // RET
    {0, 1},  // PUSH
    {1, 0},  // POP
    {1, 2},  // DUP
    {0, 1},  // LOAD
    {1, 0},  // STORE
    {0, 0},  // JMP
    {1, 0},  // JZ
    {1, 0},  // JNZ
    {2, 1}, {2, 1}, {2, 1},            // ADD SUB MUL
    {2, 1}, {2, 1},                       // FLOORDIV MOD
    {2, 1}, {2, 1}, {2, 1}, {2, 1}, {2, 1}, {2, 1},   // EQ .. GE
    {1, 1}, {1, 1},                       // NEG NOT
    {4, 1},  // EQ2
    {1, 1},  // IN (+ its values)
    {0, 1},  // ACTION
    {0, 1},  // FRAME
    {0, 1},  // FIELD
    {0, 1},  // GETR
    {1, 0},  // SETR
    {0, 1},  // GETP
    {1, 0},  // SETP
    {2, 1},  // BOARD
    {2, 1},  // BACKDROP
    {2, 1},  // CURTAIN
    {3, 0},  // SETCELL
    {1, 0},  // FILL
    {0, 1},  // ANY
    {0, 1},  // MOVE
    {2, 0},  // TELEPORT
    {1, 0},  // REWARD
    {0, 0},  // REWARD_F64
    {0, 0},  // TERMINATE
    {0, 0},  // DISCOUNT
    {2, 1},  // RANDINT
    {0, 1},  // RANDCMP
    {1, 1},  // PICK (+ its values)
    {0, 0},  // SCROLL
    {2, 2},  // PRESCROLL
    {2, 2},  // POSTSCROLL
    {2, 1},  // PATTERN
    {3, 0},  // SETPAT
    {0, 1},  // PATANY
    {1, 0},  // SETFIELD
    {3, 0},  // SETBACK
    {1, 0},  // FILLBACK
    {1, 0},  // ROLLBACK
};
static_assert(sizeof(kOps) / sizeof(kOps[0]) == PCL_OP_COUNT, "one kOps entry per opcode");
constexpr int kMaxIn = 64;            // values of an IN or a PICK

// Python's // and % (floor semantics) on int32 operands, b != 0.
__device__ __forceinline__ int floordiv(int a, int b) {
  const long long q = (long long)a / b, r = (long long)a % b;
  return (int)((r != 0 && ((r < 0) != (b < 0))) ? q - 1 : q);
}
__device__ __forceinline__ int floormod(int a, int b) {
  const long long r = (long long)a % b;
  return (int)((r != 0 && ((r < 0) != (b < 0))) ? r + b : r);
}

// NumPy's rule for one index into an axis of n cells: one negative wrap, else in range.
__device__ __forceinline__ bool cell_index(int& i, int n) {
  if (i < 0) i += n;
  return (unsigned)i < (unsigned)n;
}

// Does a visible plain sprite (program_arg[3]) stand off the board, so that upstream's
// render, `board[tuple(position)] = ...` (rendering.py:139), raises IndexError?
// Lane s checks sprite s.
__device__ __forceinline__ bool plain_sprite_off_board(const Ctx& c) {
  const StepParams& p = *c.p;
  const int s = c.lane;
  bool off = false;
  if (s < p.S && ((p.program_arg[3] >> s) & 1)) {
    const int32_t* rec = c.st->sprites[s];
    int r = rec[PCL_S_ROW], col = rec[PCL_S_COL];
    off = (rec[PCL_S_FLAGS] & 1) && !(cell_index(r, p.H) && cell_index(col, p.W));
  }
  return __any_sync(PCL_FULL, off);
}

// Valid curtain bits of word w of a bit row of W cells.
__device__ __forceinline__ uint32_t row_word_mask(int w, int W) {
  const int first = w * 32;
  if (first >= W) return 0u;
  return W - first >= 32 ? 0xffffffffu : (1u << (W - first)) - 1u;
}

// Scrolly d's whole pattern in the env being stepped: per env when the code writes it
// (program_arg[2] bit d), else static per level.  Not read through __ldg: the same launch
// may write it.
__device__ __forceinline__ uint32_t* pattern_of(const Ctx& c, int d) {
  const StepParams& p = *c.p;
  const int64_t at = ((p.program_arg[2] >> d) & 1) ? (int64_t)c.env : c.lvl;
  return p.st.d_pattern[d] + at * p.st.pattern_bstride[d];
}

// Word w of row r of Scrolly d's pattern window at its corner: curtain cells 32w .. 32w + 31
// (pattern rows carry two zero words past the last column, so the second load stays in
// the row).
__device__ __forceinline__ uint32_t window_word(const Ctx& c, int d, int r, int w) {
  const StepParams& p = *c.p;
  const int32_t* rec = c.st->drapes[d];
  const uint32_t* row = pattern_of(c, d) + (int64_t)(rec[PCL_D_CORNER_R] + r) * p.PWW;
  const int col = rec[PCL_D_CORNER_C] + 32 * w;
  return __funnelshift_r(row[col >> 5], row[(col >> 5) + 1], col & 31) & row_word_mask(w, p.W);
}

// Word w of row r of drape d's curtain: its bits, or a Scrolly's window (drapes.py:689-695).
__device__ __forceinline__ uint32_t curtain_word(const Ctx& c, int d, int r, int w) {
  if (c.p->drape_kind[d] && !((c.kept >> d) & 1)) return window_word(c, d, r, w);
  return board::bits_row(c, d, r)[w];
}

// RNG slot `slot` of the env being stepped: d_rng is u32 [B, program_arg[1], PCL_MT_WORDS].
__device__ __forceinline__ uint32_t* rng_slot(const Ctx& c, int slot) {
  const StepParams& p = *c.p;
  return p.st.d_rng + ((int64_t)c.env * p.program_arg[1] + slot) * PCL_MT_WORDS;
}

// `x cmp y` for cmp 0-5 = == != < <= > >= (PCL_OP_EQ .. PCL_OP_GE in order).
template <typename T>
__device__ __forceinline__ int compare(int cmp, T x, T y) {
  switch (cmp) {
    case 0: return x == y;
    case 1: return x != y;
    case 2: return x < y;
    case 3: return x <= y;
    case 4: return x > y;
    default: return x >= y;
  }
}

// A motion helper of Scrolly d (drapes.py:487-659).  Every path ends in _update_curtain, so
// a Scrolly whose curtain is kept in d_bits copies its new window there; the others are
// read from their static pattern at their corner, which only this call moves.
__device__ __forceinline__ void scroll(const Ctx& c, int d, int motion, Plot& plot) {
  board::scrolly_move_dyn(c, d, motion, plot);
  if ((c.kept >> d) & 1) {
    const StepParams& p = *c.p;
    for (int i = c.lane; i < p.H * p.BW; i += 32) {
      const int r = i / p.BW, w = i - r * p.BW;
      board::bits_row(c, d, r)[w] = window_word(c, d, r, w);
    }
    __syncwarp();
  }
}

struct Rewards {
  int has;
  int sum_i;
  double sum_f;
};

// The twist of a draw, out of line: inlined into the interpreter it makes ptxas spill to
// local memory.  Only one output in 624 pays for the call.
__device__ __noinline__ void twist_out_of_line(uint32_t* mt, int lane) { mt_twist(mt, lane); }

// Rotate the band of cells of rows lo .. hi - 1 of `bd` as np.roll(band, shift, axis) does:
// along each row (axis 1) or across whole rows (axis 0), by three reversals (all of it, then
// its first k and its last n - k cells, k = shift mod n), with the warp's lanes swapping
// pairs and a __syncwarp between reversals.
__device__ void roll_band(uint8_t* bd, int pitch, int W, int axis, int lo, int hi, int shift,
                          int lane) {
  const int n = axis ? W : hi - lo;          // cells along the axis
  const int lines = axis ? hi - lo : W;      // rows (axis 1) or columns (axis 0) rolled
  if (n <= 1 || lines <= 0) return;
  const int k = (int)(((long long)shift % n + n) % n);
  if (k == 0) return;
  for (int s = 0; s < 3; ++s) {                // [0, n), then [0, k), then [k, n)
    const int a = s == 2 ? k : 0, len = (s == 1 ? k : n) - a, half = len / 2;
    for (int i = lane; i < half * lines; i += 32) {
      const int line = i / half, j = i - line * half;
      const int x = a + j, y = a + len - 1 - j;
      uint8_t* u = axis ? bd + (int64_t)(lo + line) * pitch + x : bd + (int64_t)(lo + x) * pitch + line;
      uint8_t* v = axis ? bd + (int64_t)(lo + line) * pitch + y : bd + (int64_t)(lo + y) * pitch + line;
      const uint8_t t = *u;
      *u = *v;
      *v = t;
    }
    __syncwarp();
  }
}

// PCL_OP_SETBACK (x, y, v = r, c, value), FILLBACK (x = value) and ROLLBACK (a = axis, lo, hi,
// x = shift) on `bd`, the env's live curtain of H x W cells.  Only backdrop_step runs them.
// False: SETBACK's cell is off the board (nothing written).
__device__ __forceinline__ bool write_backdrop(uint8_t* bd, int H, int W, int pitch, int lane, int op,
                                            int a, int lo, int hi, int x, int y, int v) {
  __syncwarp();                              // every lane has read what it is about to change
  if (op == PCL_OP_SETBACK) {
    if (!(cell_index(x, H) && cell_index(y, W))) return false;
    if (lane == 0) bd[(int64_t)x * pitch + y] = (uint8_t)v;
  } else if (op == PCL_OP_FILLBACK) {
    for (int i = lane; i < H * W; i += 32) {
      const int r = i / W;
      bd[(int64_t)r * pitch + (i - r * W)] = (uint8_t)x;
    }
  } else {
    roll_band(bd, pitch, W, a, lo, hi, x, lane);
  }
  __syncwarp();
  return true;
}

// The update() of entity `ent` (sprites first, then drapes; S + D is the Backdrop).  kDraws:
// the code may draw (program_arg[1] > 0); games without draws run a kernel without the
// generator.  kScroll:
// the game scrolls (has Scrollys or egocentric walkers); the others run a kernel without
// the Scrolly motion helper and egocentric moves, which cost ptxas 23 more registers.
// kBackdrop: the game has a compiled Backdrop (program_arg[4]); only backdrop_step runs its
// opcodes, so compiled_step keeps the registers it had without them.
template <bool kDraws, bool kScroll, bool kBackdrop>
__device__ void run_update(const Ctx& c, Vm* vm, int ent, int action, Plot& plot,
                           Directives& dir, Rewards& rw) {
  const StepParams& p = *c.p;
  WarpState* st = c.st;
  const int S = p.S, H = p.H, W = p.W, lane = c.lane;
  const int32_t* code = p.code;
  const bool is_sprite = ent < S;
  // Registers: a walker's AUX0-AUX2 (an egocentric one's permits fill AUX0 / AUX1), a plain
  // sprite's VROW, VCOL and AUX0-AUX2 (register k >= `hole` skips FLAGS), a Scrolly's
  // AUX0-AUX2, a plain drape's whole record.
  const bool plain = is_sprite && ((p.program_arg[3] >> ent) & 1);
  const int hole = plain ? PCL_S_FLAGS - PCL_S_VROW : PCL_SPRITE_WORDS;
  int32_t* regs = is_sprite ? &st->sprites[ent][plain ? PCL_S_VROW
                                                : kScroll && p.egocentric[ent] ? PCL_S_AUX2
                                                                               : PCL_S_AUX0]
                 : kBackdrop && ent == S + p.D ? nullptr             // the Backdrop has none
                 : &st->drapes[ent - S][kScroll && p.drape_kind[ent - S] ? PCL_D_AUX0 : 0];
  const LaneSlots stk = {&vm->stack[0][lane]};
  const LaneSlots loc = {&vm->local[0][lane]};
  int sp = 0;
  int pc = __ldg(code + 1 + ent);
  for (int i = 0; i < PCL_CODE_LOCALS; ++i) loc[i] = 0;
  for (;;) {
    const int op = __ldg(code + pc);
    const int a = __ldg(code + pc + 1);      // first operand (the device copy is padded)
    int next = pc + 1 + op_operands(op);
    switch (op) {
      case PCL_OP_RET: return;
      case PCL_OP_PUSH: stk[sp++] = a; break;
      case PCL_OP_POP: --sp; break;
      case PCL_OP_DUP: stk[sp] = stk[sp - 1]; ++sp; break;
      case PCL_OP_LOAD: stk[sp++] = loc[a]; break;
      case PCL_OP_STORE: loc[a] = stk[--sp]; break;
      case PCL_OP_JMP: next = a; break;
      case PCL_OP_JZ: if (stk[--sp] == 0) next = a; break;
      case PCL_OP_JNZ: if (stk[--sp] != 0) next = a; break;
      case PCL_OP_ADD: case PCL_OP_SUB: case PCL_OP_MUL: case PCL_OP_FLOORDIV: case PCL_OP_MOD:
      case PCL_OP_EQ: case PCL_OP_NE: case PCL_OP_LT: case PCL_OP_LE: case PCL_OP_GT:
      case PCL_OP_GE: {
        const int y = stk[--sp], x = stk[sp - 1];
        const unsigned ux = (unsigned)x, uy = (unsigned)y;   // wrapping arithmetic
        int v = 0;
        switch (op) {
          case PCL_OP_ADD: v = (int)(ux + uy); break;
          case PCL_OP_SUB: v = (int)(ux - uy); break;
          case PCL_OP_MUL: v = (int)(ux * uy); break;
          case PCL_OP_FLOORDIV:
          case PCL_OP_MOD:
            if (y == 0) plot.error |= PCL_ENV_ERR_ARITH;
            else v = op == PCL_OP_MOD ? floormod(x, y) : floordiv(x, y);
            break;
          default: v = compare(op - PCL_OP_EQ, x, y); break;
        }
        stk[sp - 1] = v;
        break;
      }
      case PCL_OP_NEG: stk[sp - 1] = (int)(0u - (unsigned)stk[sp - 1]); break;
      case PCL_OP_NOT: stk[sp - 1] = stk[sp - 1] == 0; break;
      case PCL_OP_EQ2: {
        sp -= 3;
        stk[sp - 1] = stk[sp - 1] == stk[sp + 1] && stk[sp] == stk[sp + 2];
        break;
      }
      case PCL_OP_IN: {
        const int x = stk[sp - 1];
        int hit = 0;
        for (int k = 0; k < a; ++k) hit |= __ldg(code + pc + 2 + k) == x;
        stk[sp - 1] = hit;
        next += a;
        break;
      }
      case PCL_OP_ACTION: stk[sp++] = action; break;
      case PCL_OP_FRAME: stk[sp++] = plot.frame; break;
      case PCL_OP_FIELD: {
        const int32_t* rec = st->sprites[a < 0 ? ent : a];
        const int f = __ldg(code + pc + 2);
        stk[sp++] = f == 4 ? (rec[PCL_S_FLAGS] & 1) : rec[f];
        break;
      }
      case PCL_OP_GETR: stk[sp++] = regs[a + (a >= hole)]; break;
      case PCL_OP_SETFIELD: {                  // row, col or the visible bit of FLAGS
        const int v = stk[--sp];
        int32_t* rec = st->sprites[ent];
        __syncwarp();
        if (lane == 0) rec[a] = a == PCL_S_FLAGS ? (rec[a] & ~1) | (v != 0) : v;
        __syncwarp();
        break;
      }
      case PCL_OP_SETR: {
        const int v = stk[--sp];
        __syncwarp();
        if (lane == 0) regs[a + (a >= hole)] = v;
        __syncwarp();
        break;
      }
      case PCL_OP_GETP: stk[sp++] = st->plot[PCL_P_AUX0 + a]; break;
      case PCL_OP_SETP: {
        const int v = stk[--sp];
        __syncwarp();
        if (lane == 0) st->plot[PCL_P_AUX0 + a] = v;
        __syncwarp();
        break;
      }
      case PCL_OP_BOARD: case PCL_OP_BACKDROP: case PCL_OP_CURTAIN: {
        int col = stk[--sp], r = stk[sp - 1];
        int v = 0;
        if (cell_index(r, H) && cell_index(col, W)) {
          if (op == PCL_OP_BOARD) v = c.board[r * p.pitch + col];
          else if (op == PCL_OP_BACKDROP) v = c.backdrop[(int64_t)r * p.pitch + col];
          else if (kScroll) v = board::drape_bit(c, (a < 0 ? ent : a) - S, r, col);
          else v = bit_at(board::bits_row(c, (a < 0 ? ent : a) - S, r), col);
        } else {
          plot.error |= PCL_ENV_ERR_INDEX;
        }
        stk[sp - 1] = v;
        break;
      }
      case PCL_OP_SETCELL: {
        sp -= 3;
        const int v = stk[sp + 2];
        int r = stk[sp], col = stk[sp + 1];
        if (cell_index(r, H) && cell_index(col, W)) {
          uint32_t* row = board::bits_row(c, ent - S, r);
          __syncwarp();
          if (lane == 0) {
            const uint32_t bit = 1u << (col & 31);
            row[col >> 5] = v ? (row[col >> 5] | bit) : (row[col >> 5] & ~bit);
          }
          __syncwarp();
        } else {
          plot.error |= PCL_ENV_ERR_INDEX;
        }
        break;
      }
      case PCL_OP_FILL: {
        const int v = stk[--sp];
        __syncwarp();
        for (int i = lane; i < H * p.BW; i += 32) {
          const int r = i / p.BW, w = i - r * p.BW;
          board::bits_row(c, ent - S, r)[w] = v ? row_word_mask(w, W) : 0u;
        }
        __syncwarp();
        break;
      }
      case PCL_OP_ANY: {
        const int d = (a < 0 ? ent : a) - S;
        bool any = false;
        for (int i = lane; i < H * p.BW; i += 32) {
          const int r = i / p.BW, w = i - r * p.BW;
          any |= (kScroll ? curtain_word(c, d, r, w) : board::bits_row(c, d, r)[w]) != 0u;
        }
        stk[sp++] = __any_sync(PCL_FULL, any) ? 1 : 0;
        break;
      }
      case PCL_OP_MOVE: {
        Sprite s = load_sprite(st->sprites[ent]);
        const uint32_t* imp = st->impassable[ent];
        const uint8_t* bd = c.board;
        const int pitch = p.pitch;
        const bool moved = walker_move(s, ent, a, plot, H, W, p.confined[ent] != 0,
                                       kScroll && p.egocentric[ent] != 0, lane,
                                       [&](int r, int col) { return in_set(imp, bd[r * pitch + col]); });
        board::warp_store_sprite(st->sprites[ent], s, lane);
        stk[sp++] = moved ? 0 : 1;
        break;
      }
      case PCL_OP_TELEPORT: {
        sp -= 2;
        Sprite s = load_sprite(st->sprites[ent]);
        walker_teleport(s, H, W, stk[sp], stk[sp + 1]);
        board::warp_store_sprite(st->sprites[ent], s, lane);
        break;
      }
      case PCL_OP_REWARD: case PCL_OP_REWARD_F64: {
        const int x = op == PCL_OP_REWARD ? stk[--sp] : 0;
        const double f = op == PCL_OP_REWARD ? (double)x
                                             : __hiloint2double(__ldg(code + pc + 2), a);
        rw.sum_f = rw.has ? rw.sum_f + f : f;    // Python's `None`, then `reward + r`
        rw.sum_i = (int)((unsigned)rw.sum_i + (unsigned)x);
        rw.has = 1;
        break;
      }
      case PCL_OP_TERMINATE: terminate(dir, __int_as_float(a)); break;
      case PCL_OP_DISCOUNT: change_default_discount(dir, __int_as_float(a)); break;
      case PCL_OP_RANDINT: case PCL_OP_RANDCMP: {   // one mt_draw site for both
        if (!kDraws) break;                           // pcl_bind_code refused them
        const int b = __ldg(code + pc + 2);           // the rule, or the comparison
        const bool cmp = op == PCL_OP_RANDCMP;
        int low = 0;
        int64_t width = 0;
        if (!cmp) {
          const int high = stk[--sp];
          low = stk[sp - 1];
          width = (int64_t)high - low + (b == PCL_RAND_PYTHON_CLOSED);
          if (width <= 0) {                  // ValueError upstream; low stays on the stack
            plot.error |= PCL_ENV_ERR_RANGE;
            break;
          }
          --sp;
        }
        const MtRule rule = cmp ? kMtRandom53 : b == PCL_RAND_NUMPY ? kMtNumpyBelow : kMtPythonBelow;
        const uint64_t r = mt_draw<twist_out_of_line>(rng_slot(c, a), rule, (uint64_t)width, lane);
        if (cmp) {
          const double x = __dmul_rn(__ull2double_rn(r), 1.0 / 9007199254740992.0);
          stk[sp++] = compare(b, x, __hiloint2double(__ldg(code + pc + 4), __ldg(code + pc + 3)));
        } else {
          stk[sp++] = (int)((uint32_t)low + (uint32_t)r);
        }
        break;
      }
      case PCL_OP_SCROLL: if (kScroll) scroll(c, ent - S, a, plot); break;
      case PCL_OP_PRESCROLL: case PCL_OP_POSTSCROLL: {
        if (!kScroll) break;                   // pcl_bind_code refused them
        int32_t* rec = st->drapes[(a < 0 ? ent : a) - S];
        const bool stale = rec[PCL_D_LAST_FRAME] < plot.frame;
        int dr = rec[PCL_D_CORNER_R], dc = rec[PCL_D_CORNER_C];
        if (op == PCL_OP_PRESCROLL) {
          if (stale) {                         // drapes.py:407-408
            __syncwarp();
            if (lane == 0) { rec[PCL_D_PRE_R] = dr; rec[PCL_D_PRE_C] = dc; }
            __syncwarp();
          }
          dr = rec[PCL_D_PRE_R]; dc = rec[PCL_D_PRE_C];
        } else if (stale) {
          plot.error |= PCL_ENV_ERR_POSTSCROLL;   // RuntimeError upstream, drapes.py:434-438
        }
        stk[sp - 2] = (int)((unsigned)stk[sp - 2] + (unsigned)dr);
        stk[sp - 1] = (int)((unsigned)stk[sp - 1] + (unsigned)dc);
        break;
      }
      case PCL_OP_PATTERN: case PCL_OP_SETPAT: {
        if (!kScroll) break;
        const bool set = op == PCL_OP_SETPAT;
        sp -= set ? 3 : 2;
        int r = stk[sp], col = stk[sp + 1];
        const int d = (set || a < 0 ? ent : a) - S;
        int v = 0;
        if (cell_index(r, p.PH) && cell_index(col, p.PW)) {
          uint32_t* row = pattern_of(c, d) + (int64_t)r * p.PWW;
          if (set) {
            __syncwarp();
            if (lane == 0) {
              const uint32_t bit = 1u << (col & 31);
              row[col >> 5] = stk[sp + 2] ? (row[col >> 5] | bit) : (row[col >> 5] & ~bit);
            }
            __syncwarp();
          } else {
            v = bit_at(row, col);
          }
        } else {
          plot.error |= PCL_ENV_ERR_INDEX;
        }
        if (!set) stk[sp++] = v;
        break;
      }
      case PCL_OP_PATANY: {
        if (!kScroll) break;
        const uint32_t* pat = pattern_of(c, (a < 0 ? ent : a) - S);
        bool any = false;
        for (int i = lane; i < p.PH * p.PWW; i += 32) any |= pat[i] != 0u;
        stk[sp++] = __any_sync(PCL_FULL, any) ? 1 : 0;
        break;
      }
      default: {                               // PCL_OP_PICK, and the Backdrop's opcodes
        // The Backdrop's opcodes take no case labels: with them, compiled_step's dispatch
        // and register allocation would change.
        if (kBackdrop && op >= PCL_OP_SETBACK) {
          const bool set = op == PCL_OP_SETBACK, roll = op == PCL_OP_ROLLBACK;
          sp -= set ? 3 : 1;
          if (!write_backdrop(p.backdrop_live + (int64_t)c.env * H * p.pitch, H, W, p.pitch, lane, op,
                              a, roll ? __ldg(code + pc + 2) : 0, roll ? __ldg(code + pc + 3) : 0,
                              stk[sp], set ? stk[sp + 1] : 0, set ? stk[sp + 2] : 0))
            plot.error |= PCL_ENV_ERR_INDEX;
          if (roll) next += 3;                 // op_operands leaves ROLLBACK's out (code_operands)
          break;
        }
        const int i = stk[sp - 1];
        int v = 0;
        if ((unsigned)i < (unsigned)a) v = __ldg(code + pc + 2 + i);
        else plot.error |= PCL_ENV_ERR_INDEX;
        stk[sp - 1] = v;
        next += a;
        break;
      }
    }
    pc = next;
  }
}

// One env's step.  kBackdrop: as run_update; compiled_step and backdrop_step are its two
// kernels.
template <bool kDraws, bool kScroll, bool kBackdrop>
__device__ __forceinline__ void step(const StepParams& p) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int env = blockIdx.x * kWarpsPerBlock + warp;
  if (env >= p.B) return;
  const int64_t lvl = p.st.d_level ? p.st.d_level[env] : env;   // index of static level data
  const int H = p.H, S = p.S, D = p.D, n = S + D;
  const size_t board_bytes = board::board_bytes(H, p.pitch);
  uint8_t* my = smem_raw + warp * (sizeof(WarpState) + sizeof(Vm) + board_bytes);
  WarpState* st = reinterpret_cast<WarpState*>(my);
  Vm* vm = reinterpret_cast<Vm*>(my + sizeof(WarpState));
  Ctx c;
  c.p = &p; c.st = st; c.board = my + sizeof(WarpState) + sizeof(Vm);
  // A compiled Backdrop (program_arg[4]) writes its own live copy; the template is per level.
  const uint8_t* backdrop_init = p.st.d_backdrop + lvl * p.st.backdrop_bstride;
  c.backdrop = kBackdrop ? p.backdrop_live + (int64_t)env * H * p.pitch : backdrop_init;
  c.env = env; c.lane = lane; c.lvl = lvl;
  c.kept = (uint32_t)p.program_arg[2];       // Scrollys that write their pattern

  int32_t* g_sprites = p.st.d_sprites + (int64_t)env * S * PCL_SPRITE_WORDS;
  int32_t* g_drapes = p.st.d_drapes + (int64_t)env * D * PCL_DRAPE_WORDS;
  int32_t* g_plot = p.st.d_plot + (int64_t)env * PCL_PLOT_WORDS;
  uint8_t* g_z = p.st.d_z_order + (int64_t)env * n;
  uint8_t* g_board = p.out.d_board + (int64_t)env * H * p.pitch;

  const EnvRun run = env_run(p, env, g_plot[PCL_P_GAME_OVER]);
  if (run == ENV_SKIP) return;
  const bool restart = run == ENV_RESTART;
  const PlotCarry carry = plot_carry(g_plot, restart);
  board::stage_records(
      st, restart ? p.st.d_sprites_init + lvl * p.st.sprites_init_bstride : g_sprites,
      restart ? p.st.d_drapes_init + lvl * p.st.drapes_init_bstride : g_drapes,
      restart ? p.st.d_plot_init + lvl * p.st.plot_init_bstride : g_plot,
      restart ? p.st.d_z_order_init + lvl * p.st.z_order_init_bstride : g_z, S, D, lane);
  for (int i = lane; i < S * 4; i += 32) (&st->impassable[0][0])[i] = p.impassable[i >> 2][i & 3];
  if (restart) {
    // A restart rebuilds every curtain kept in bits from its template (things.py:146-217),
    // and every pattern the code writes.
    for (int d = 0; d < D; ++d) {
      if ((c.kept >> d) & 1) {
        const uint32_t* src = p.st.d_pattern_init[d] + lvl * p.st.pattern_init_bstride[d];
        uint32_t* dst = p.st.d_pattern[d] + (int64_t)env * p.st.pattern_bstride[d];
        for (int i = lane; i < p.PH * p.PWW; i += 32) dst[i] = src[i];
      }
      if (p.drape_kind[d] && !((c.kept >> d) & 1)) continue;
      const uint32_t* src = p.st.d_bits_init[d] + lvl * p.st.bits_init_bstride[d];
      uint32_t* dst = p.st.d_bits[d] + (int64_t)env * p.st.bits_bstride[d];
      for (int i = lane; i < H * p.BW; i += 32) dst[i] = src[i];
    }
    if (kBackdrop) {                         // the Backdrop's curtain, before the first render
      const uint4* src = reinterpret_cast<const uint4*>(backdrop_init);
      uint4* dst = reinterpret_cast<uint4*>(p.backdrop_live + (int64_t)env * H * p.pitch);
      for (int i = lane; i < (H * p.pitch) >> 4; i += 32) dst[i] = src[i];
    }
  }
  __syncwarp();
  if (restart) {
    if (lane == 0) store_carry(st->plot, carry);
    __syncwarp();
  }
  // Zero the board's pitch padding too: the whole H * pitch plane goes out to d_board.
  for (int i = lane; i < (int)board_bytes; i += 32) c.board[i] = 0;
  __syncwarp();
  board::stage_board</*kWrap=*/true>(c, restart, g_board);

  Plot plot = step_plot</*kOrder=*/true>(st->plot, carry.error);
  Directives dir = fresh_directives();
  Rewards rw = {0, 0, 0.0};
  const int action = restart ? PCL_ACTION_NONE : p.actions[(int64_t)env * p.actions_per_env];

  // ---- update groups (engine.py:725-735)
  int k = 0;
  if (kBackdrop) {
    // The Backdrop's update() first, as "group -1": on the board of the last render, with no
    // render after it (engine.py:718-723).  One run_update call site serves it and the
    // entities, which keeps backdrop_step free of a stack.
    for (int g = -1; g < p.n_groups; ++g) {
      for (int e = 0; e < (g < 0 ? 1 : p.group_len[g]); ++e) {
        int ent = n;
        if (g >= 0) {
          const int ch = p.group_chars[k++];
          ent = 0;
          for (int s = 0; s < S; ++s) if (p.sprite_char[s] == ch) ent = s;
          for (int d = 0; d < D; ++d) if (p.drape_char[d] == ch) ent = S + d;
        }
        run_update<kDraws, kScroll, kBackdrop>(c, vm, ent, action, plot, dir, rw);
      }
      if (g < 0) continue;
      board::render</*kWrap=*/true>(c);
      if (p.program_arg[3] && plain_sprite_off_board(c)) plot.error |= PCL_ENV_ERR_INDEX;
    }
  } else {
    for (int g = 0; g < p.n_groups; ++g) {
      for (int e = 0; e < p.group_len[g]; ++e, ++k) {
        const int ch = p.group_chars[k];
        int ent = 0;
        for (int s = 0; s < S; ++s) if (p.sprite_char[s] == ch) ent = s;
        for (int d = 0; d < D; ++d) if (p.drape_char[d] == ch) ent = S + d;
        run_update<kDraws, kScroll, kBackdrop>(c, vm, ent, action, plot, dir, rw);
      }
      board::render</*kWrap=*/true>(c);
      if (p.program_arg[3] && plain_sprite_off_board(c)) plot.error |= PCL_ENV_ERR_INDEX;
    }
  }

  __syncwarp();
  if (lane == 0) {
    const double ep_so_far = load_episode(p, env);   // overlaps the stores below
    apply_time_limit(p, plot, dir);
    store_episode(p, env, plot.frame, ep_so_far, p.program_arg[0] ? (rw.has ? rw.sum_f : 0.0) : (double)(rw.has ? rw.sum_i : 0));
    store_plot<ORDER_ALL>(st->plot, plot, dir);
    dir.reward = rw.has ? rw.sum_i : 0; dir.has_reward = rw.has;   // the code's own sums
    if (p.program_arg[0]) store_outputs(p.out, env, dir, rw.has ? rw.sum_f : 0.0);
    else store_outputs(p.out, env, dir);
  }
  __syncwarp();
  board::store_env(c, g_sprites, g_drapes, g_plot, g_z, g_board);
}

template <bool kDraws, bool kScroll>
__global__ void __launch_bounds__(kWarpsPerBlock * 32) compiled_step(const StepParams p) {
  step<kDraws, kScroll, false>(p);
}

// Games whose Backdrop has compiled update() code (program_arg[4]).
template <bool kDraws, bool kScroll>
__global__ void __launch_bounds__(kWarpsPerBlock * 32) backdrop_step(const StepParams p) {
  step<kDraws, kScroll, true>(p);
}

// MazeWalkers, plain Sprites, Scrollys and plain drapes in one scrolling group; the entities and the
// z-order are consistent permutations of each other.
int check_spec(const pcl_spec& s) {
  const int n = s.n_sprites + s.n_drapes;
  if (n < 1) return PCL_ERR_INVALID;
  if (s.n_groups < 1 || s.n_groups > board::kMaxEnt) return PCL_ERR_INVALID;
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
    if (s.drape_kind[d] != 0 && s.drape_kind[d] != 1) return PCL_ERR_UNSUPPORTED;
    if (!s.drape_kind[d]) continue;
    if (s.pattern_rows < s.rows || s.pattern_cols < s.cols) return PCL_ERR_INVALID;
    if (s.pattern_words < (s.pattern_cols + 31) / 32 + 2) return PCL_ERR_INVALID;
    if (!margins_fit(s, d)) return PCL_ERR_INVALID;
  }
  if (s.program_arg[0] != 0 && s.program_arg[0] != 1) return PCL_ERR_INVALID;
  if (s.program_arg[1] < 0 || s.program_arg[1] > 2) return PCL_ERR_INVALID;   // RNG slots
  // Written patterns: Scrollys only.
  const uint32_t kept = (uint32_t)s.program_arg[2];
  for (int d = 0; d < 32; ++d)
    if (((kept >> d) & 1) && (d >= s.n_drapes || !s.drape_kind[d])) return PCL_ERR_INVALID;
  // Plain Sprites: sprites only, and not egocentric.
  const uint32_t plain = (uint32_t)s.program_arg[3];
  for (int i = 0; i < 32; ++i)
    if (((plain >> i) & 1) && (i >= s.n_sprites || s.sprite_egocentric[i])) return PCL_ERR_INVALID;
  if (s.program_arg[4] != 0 && s.program_arg[4] != 1) return PCL_ERR_INVALID;   // a compiled Backdrop
  if (!bit_rows_fit(s)) return PCL_ERR_INVALID;
  return PCL_OK;
}

int check_state(const pcl_spec& s, const pcl_state& st) {
  if (!st.d_z_order || !st.d_z_order_init) return PCL_ERR_INVALID;
  for (int d = 0; d < s.n_drapes; ++d) {
    const bool kept = (s.program_arg[2] >> d) & 1;
    if (s.drape_kind[d] && !st.d_pattern[d]) return PCL_ERR_INVALID;
    if (kept && (!st.d_pattern_init[d] || st.pattern_bstride[d] == 0)) return PCL_ERR_INVALID;
    if ((!s.drape_kind[d] || kept) && (!st.d_bits[d] || !st.d_bits_init[d])) return PCL_ERR_INVALID;
  }
  if (s.program_arg[1] > 0 && !st.d_rng) return PCL_ERR_INVALID;
  return PCL_OK;
}

int rng_slots(const pcl_spec& s) { return s.program_arg[1]; }

// Scrollys' curtains: kept in bits when their pattern is written, else their window.
CurtainAt curtain(const pcl_spec& s, int d) {
  return s.drape_kind[d] && !((s.program_arg[2] >> d) & 1) ? CurtainAt::kPatternWindow
                                                            : CurtainAt::kBits;
}

// The checks pcl_bind_code promises (include/pcl.h): after them the kernel can run any
// entity's code without a bounds test.
int check_code(const pcl_spec& s, const int32_t* w, int n) {
  // With a compiled Backdrop, header word 1 + ents is its function's entry.
  const bool has_backdrop = s.program_arg[4] != 0;
  const int S = s.n_sprites, ents = s.n_sprites + s.n_drapes, body = 1 + ents + has_backdrop;
  if (n <= body || n > PCL_MAX_CODE_WORDS || w[0] != ents) return PCL_ERR_INVALID;
  // A walker, a plain Sprite and the Backdrop are different kinds: their functions take
  // different opcodes.
  enum { kNone = 0, kSprite = 1, kDrape = 2, kPlainSprite = 3, kBackdrop = 4 };
  const uint32_t plain_sprites = (uint32_t)s.program_arg[3];
  auto is_plain_sprite = [&](int k) { return k >= 0 && k < S && ((plain_sprites >> k) & 1); };
  // What the entities sharing a function allow it: their kind, the fewest registers any of
  // them has (1 for an egocentric walker, 3 for a walker or a Scrolly, 5 for a plain
  // sprite, 8 for a plain drape), whether they are all Scrollys, all plain drapes, all
  // Scrollys that write their pattern.
  struct Fn { int8_t kind, regs; bool scrolly, plain, writes; };
  std::vector<Fn> starts(n, Fn{kNone, 0, false, false, false});   // by first word
  for (int i = 0; i < ents; ++i) {
    const int e = w[1 + i];
    const int kind = i >= S ? kDrape : is_plain_sprite(i) ? kPlainSprite : kSprite;
    if (e < body || e >= n) return PCL_ERR_INVALID;
    if (starts[e].kind != kNone && starts[e].kind != kind) return PCL_ERR_INVALID;
    const bool scrolly = kind == kDrape && s.drape_kind[i - S];
    const bool writes = scrolly && ((s.program_arg[2] >> (i - S)) & 1);
    const int regs = kind == kPlainSprite ? 5
                     : kind == kSprite ? (s.sprite_egocentric[i] ? 1 : 3)
                                       : (scrolly ? 3 : PCL_DRAPE_WORDS);
    Fn& f = starts[e];
    if (f.kind == kNone) f = Fn{(int8_t)kind, (int8_t)regs, scrolly, !scrolly && kind == kDrape, writes};
    f.regs = (int8_t)(regs < f.regs ? regs : f.regs);
    f.scrolly = f.scrolly && scrolly;
    f.plain = f.plain && !scrolly && kind == kDrape;
    f.writes = f.writes && writes;
  }
  if (has_backdrop) {                          // no registers, and a function of its own
    const int e = w[1 + ents];
    if (e < body || e >= n || starts[e].kind != kNone) return PCL_ERR_INVALID;
    starts[e] = Fn{kBackdrop, 0, false, false, false};
  }
  if (starts[body].kind == kNone) return PCL_ERR_INVALID;
  // An entity operand naming a Scrolly, or -1 in a function of Scrollys.
  auto is_scrolly = [&](int a, const Fn& f) {
    return a < 0 ? f.scrolly : (a >= S && a < ents && s.drape_kind[a - S] != 0);
  };
  std::vector<int> depth(n, -1);                 // stack depth on arrival, -1 = unreachable
  std::vector<int8_t> boundary(n, 0);
  std::vector<int> targets;
  int kind = kNone, end = 0;
  Fn fn = starts[body];
  for (int pc = body; pc < n;) {
    if (starts[pc].kind != kNone) {              // a new function
      fn = starts[pc];
      kind = fn.kind;
      for (end = pc + 1; end < n && starts[end].kind == kNone; ++end) {}
      depth[pc] = 0;
    }
    boundary[pc] = 1;
    const int op = w[pc];
    if (op < 0 || op >= PCL_OP_COUNT) return PCL_ERR_INVALID;
    int len = 1 + code_operands(op);
    if (pc + len > end) return PCL_ERR_INVALID;
    const int a = len > 1 ? w[pc + 1] : 0;
    const bool walker = kind == kSprite, plain_sprite = kind == kPlainSprite;
    const bool sprite = walker || plain_sprite, backdrop = kind == kBackdrop;
    switch (op) {
      case PCL_OP_LOAD: case PCL_OP_STORE:
        if (a < 0 || a >= PCL_CODE_LOCALS) return PCL_ERR_INVALID;
        break;
      case PCL_OP_JMP: case PCL_OP_JZ: case PCL_OP_JNZ:
        if (a <= pc || a >= end) return PCL_ERR_INVALID;
        targets.push_back(a);
        break;
      case PCL_OP_IN: case PCL_OP_PICK:
        if (a < (op == PCL_OP_PICK ? 1 : 0) || a > kMaxIn) return PCL_ERR_INVALID;
        len += a;
        if (pc + len > end) return PCL_ERR_INVALID;
        break;
      case PCL_OP_RANDINT:
        if (a < 0 || a >= s.program_arg[1]) return PCL_ERR_INVALID;
        if (w[pc + 2] < PCL_RAND_NUMPY || w[pc + 2] > PCL_RAND_PYTHON_CLOSED) return PCL_ERR_INVALID;
        break;
      case PCL_OP_RANDCMP:
        if (a < 0 || a >= s.program_arg[1]) return PCL_ERR_INVALID;
        if (w[pc + 2] < 0 || w[pc + 2] > 5) return PCL_ERR_INVALID;
        break;
      case PCL_OP_FIELD: {
        if (a < 0 ? !sprite : a >= S) return PCL_ERR_INVALID;
        const int f = w[pc + 2];
        if (f < 0 || f > 4) return PCL_ERR_INVALID;
        // A plain Sprite has no virtual position.
        if ((f == PCL_S_VROW || f == PCL_S_VCOL) && (a < 0 ? plain_sprite : is_plain_sprite(a)))
          return PCL_ERR_INVALID;
        break;
      }
      case PCL_OP_SETFIELD:
        if (!plain_sprite || (a != PCL_S_ROW && a != PCL_S_COL && a != PCL_S_FLAGS))
          return PCL_ERR_INVALID;
        break;
      case PCL_OP_GETR: case PCL_OP_SETR:
        if (a < 0 || a >= fn.regs) return PCL_ERR_INVALID;
        break;
      case PCL_OP_GETP: case PCL_OP_SETP:
        if (a < 0 || a >= 4) return PCL_ERR_INVALID;
        break;
      case PCL_OP_CURTAIN: case PCL_OP_ANY:
        if (a < 0 ? sprite || backdrop : (a < S || a >= ents)) return PCL_ERR_INVALID;
        break;
      case PCL_OP_SETBACK: case PCL_OP_FILLBACK:
        if (!backdrop) return PCL_ERR_INVALID;
        break;
      case PCL_OP_ROLLBACK:
        if (!backdrop || (a != 0 && a != 1)) return PCL_ERR_INVALID;
        if (w[pc + 2] < 0 || w[pc + 2] > w[pc + 3] || w[pc + 3] > s.rows) return PCL_ERR_INVALID;
        break;
      case PCL_OP_SETCELL: case PCL_OP_FILL:
        if (!fn.plain) return PCL_ERR_INVALID;   // a Scrolly's curtain is its pattern's window
        break;
      case PCL_OP_SCROLL:
        if (!fn.scrolly || a < 0 || a > PCL_M_STAY) return PCL_ERR_INVALID;
        break;
      case PCL_OP_SETPAT:
        if (!fn.scrolly || !fn.writes) return PCL_ERR_INVALID;
        break;
      case PCL_OP_PRESCROLL: case PCL_OP_POSTSCROLL: case PCL_OP_PATTERN: case PCL_OP_PATANY:
        if (!is_scrolly(a, fn)) return PCL_ERR_INVALID;
        break;
      case PCL_OP_MOVE:
        if (!walker || a < 0 || a > PCL_M_STAY) return PCL_ERR_INVALID;
        break;
      case PCL_OP_TELEPORT:
        if (!walker) return PCL_ERR_INVALID;
        break;
      case PCL_OP_REWARD_F64:
        if (!s.program_arg[0]) return PCL_ERR_INVALID;   // an int32 reward cannot carry it
        break;
      default: break;
    }
    const int d = depth[pc];
    if (d >= 0) {
      if (d < kOps[op].pops) return PCL_ERR_INVALID;
      const int after = d - kOps[op].pops + kOps[op].pushes;
      if (after > PCL_CODE_STACK) return PCL_ERR_INVALID;
      auto arrive = [&](int t) {
        if (depth[t] >= 0 && depth[t] != after) return false;
        depth[t] = after;
        return true;
      };
      if ((op == PCL_OP_JMP || op == PCL_OP_JZ || op == PCL_OP_JNZ) && !arrive(a))
        return PCL_ERR_INVALID;
      if (op != PCL_OP_RET && op != PCL_OP_JMP) {
        if (pc + len >= end) return PCL_ERR_INVALID;   // falls off the end of its function
        if (!arrive(pc + len)) return PCL_ERR_INVALID;
      }
    }
    pc += len;
  }
  for (int t : targets)
    if (!boundary[t]) return PCL_ERR_INVALID;
  return PCL_OK;
}

int actions_per_env(const pcl_spec&) { return 1; }

cudaError_t launch(const StepParams& p, cudaStream_t s) {
  const size_t smem = (sizeof(WarpState) + sizeof(Vm) + board::board_bytes(p.H, p.pitch)) *
                      kWarpsPerBlock;
  bool scrolls = false;
  for (int d = 0; d < p.D; ++d) scrolls = scrolls || p.drape_kind[d];
  for (int i = 0; i < p.S; ++i) scrolls = scrolls || p.egocentric[i];
  const bool draws = p.program_arg[1] > 0;
  if (p.program_arg[4]) {
    if (scrolls)
      return draws ? launch_step(backdrop_step<true, true>, p, kWarpsPerBlock, smem, s)
                   : launch_step(backdrop_step<false, true>, p, kWarpsPerBlock, smem, s);
    return draws ? launch_step(backdrop_step<true, false>, p, kWarpsPerBlock, smem, s)
                 : launch_step(backdrop_step<false, false>, p, kWarpsPerBlock, smem, s);
  }
  if (scrolls)
    return draws ? launch_step(compiled_step<true, true>, p, kWarpsPerBlock, smem, s)
                 : launch_step(compiled_step<false, true>, p, kWarpsPerBlock, smem, s);
  return draws ? launch_step(compiled_step<true, false>, p, kWarpsPerBlock, smem, s)
               : launch_step(compiled_step<false, false>, p, kWarpsPerBlock, smem, s);
}

}  // namespace

const Program kCompiled = {check_spec, check_state, curtain, launch, actions_per_env,
                           /*float_reward=*/false, /*crop_epilogue=*/false,
                           /*scroll_groups=*/false, check_code, /*float_reward_arg0=*/true,
                           /*derive=*/nullptr, /*block_chaining=*/false, rng_slots};

}  // namespace pcl
