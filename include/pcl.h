/*
 * pcl.h — C ABI of the H100 batched gridworld step engine (libpcl.so).
 *
 * pycolab has no FFI: its "plugin interface" for the per-step hot path is the
 * Python object API  Engine.its_showtime() / Engine.play(actions)  returning
 * (Observation(board, layers), reward, discount)  (reference
 * pycolab/engine.py:520-639).  This header is what a native replacement of
 * that path exports; INTEGRATION.md shows the ctypes binding a pycolab
 * maintainer would add.  Conventions (SURVEY.md §8b):
 *
 *   - plain C, no C++/torch types; every pointer named d_* is a DEVICE
 *     pointer, h_* a HOST pointer; buffers are owned by the caller, the
 *     library never frees them;
 *   - every entry point returns 0 (PCL_OK) or a negative pcl_status and never
 *     throws; per-environment run-time faults (the reference's RuntimeError /
 *     scrolling.Error cases) are latched in a per-env error word readable
 *     with pcl_error_codes();
 *   - every launch takes the cudaStream_t (as void*) to enqueue on; nothing
 *     synchronises except the *_host entry points;
 *   - re-entrant per handle, no global state.
 *
 * Batched-state model: B independent environments ("envs"), each the
 * equivalent of one reference Engine, live as a struct-of-arrays in HBM.
 * One warp advances one env per launch.
 */
#ifndef PCL_H_
#define PCL_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PCL_ABI_VERSION 3

#define PCL_MAX_SPRITES 16
#define PCL_MAX_DRAPES 8
#define PCL_SPRITE_WORDS 8   /* int32 words per sprite record */
#define PCL_DRAPE_WORDS 8    /* int32 words per drape record  */
#define PCL_PLOT_WORDS 16    /* int32 words per env plot record */
#define PCL_MT_WORDS 625     /* MT19937: 624 state words + position */
#define PCL_MAX_SCROLL_GROUPS 4 /* scrolling groups of one game (protocols/scrolling.py:198-241) */
#define PCL_GROUP_WORDS 4    /* int32 words per scrolling-group record */

typedef enum pcl_status {
  PCL_OK = 0,
  PCL_ERR_INVALID = -1,      /* bad argument / malformed spec (ValueError)   */
  PCL_ERR_UNSUPPORTED = -2,  /* spec is valid pycolab but not lowered        */
  PCL_ERR_CUDA = -3,         /* a CUDA runtime call failed                   */
  PCL_ERR_UNBOUND = -4,      /* pcl_bind_state (or pcl_bind_code) has not been called */
  PCL_ERR_NOMEM = -5
} pcl_status;

/* Per-env latched error bits (pcl_error_codes).  Each mirrors an exception
 * the reference would raise inside Engine.play(). */
#define PCL_ENV_ERR_ORDER_MISMATCH   0x1  /* sprites.py:449-454, drapes.py:525-530 */
#define PCL_ENV_ERR_SECOND_ORDER     0x2  /* scrolling.py:518-521 */
#define PCL_ENV_ERR_EMPTY_CHOICE     0x4  /* np.random.choice([]) in marauders :253 */
#define PCL_ENV_ERR_INDEX            0x8  /* NumPy IndexError (board look-up off the array) */
#define PCL_ENV_ERR_BAD_Z            0x10 /* change_z_order names a missing entity, engine.py:802-812 */
#define PCL_ENV_ERR_ARITH            0x20 /* ZeroDivisionError: `//` or `%` by zero in compiled code */
#define PCL_ENV_ERR_RANGE            0x40 /* ValueError: a compiled draw from an empty range */
#define PCL_ENV_ERR_POSTSCROLL       0x80 /* pattern_position_postscroll before the Scrolly moved, drapes.py:434-438 */

/* Which game program advances the envs.  One fused kernel per program; the
 * host "lowering" recognises the reference's entity classes and picks one. */
typedef enum pcl_program {
  PCL_PROG_NONE = 0,         /* no step program: pcl_render / pcl_crop only        */
  PCL_PROG_SCROLLY_MAZE = 1, /* examples/scrolly_maze.py:212-364               */
  PCL_PROG_WAREHOUSE = 2,    /* examples/warehouse_manager.py:139-295          */
  PCL_PROG_MARAUDERS = 3,    /* examples/extraterrestrial_marauders.py:91-256  */
  PCL_PROG_FIXTURE = 4,      /* tests/test_things.py TestMazeWalker/TestScrolly */
  PCL_PROG_BETTER_SCROLLY = 5, /* examples/better_scrolly_maze.py:209-324       */
  PCL_PROG_CLASSICS = 6,     /* one-walker games: examples/classics/{four_rooms,cliff_walk,
                                chain_walk}.py, examples/fluvial_natation.py */
  PCL_PROG_APERTURE = 7,     /* examples/aperture.py:118-196; the drape record's AUX0 / AUX1 hold
                                the two aperture cells (row << 16 | col, -1 = none) */
  PCL_PROG_HELLO = 9,        /* examples/hello_world.py:58-118: plain Sprites (aux0 = direction set)
                                + one rolling Drape (record AUX0 / AUX1 = row / column shift of the
                                reset curtain); program_arg[0..n) = the z-order chars */
  PCL_PROG_APPREHEND = 10,   /* examples/apprehend.py:56-131: sprites 'P' (confined catcher) and 'b' (falling
                                ball); the ball's AUX0 / AUX1 hold its float64 slope (bits lo / hi), plot
                                AUX0 / AUX1 its x accumulator; with pcl_state.d_rng bound (the words of
                                Python's random.Random(seed).getstate()) the slope is drawn on the device at
                                every (re)start as random.uniform does, else taken from the reset template */
  PCL_PROG_SHOCKWAVE = 11,   /* examples/shockwave.py:91-197: sprite 'P', drapes '@' (curtain bit-packed in
                                d_bits[0], record AUX0 = impact cell index, AUX1 = steps since impact), ' '
                                and '^' (static, d_bits_init[1..2]); program_arg[0] = ring width; d_rng =
                                NumPy RandomState words (np.random.randint picks the impact cell) */
  PCL_PROG_T_MAZE = 12,      /* examples/research/lp-rnn/t_maze.py:180-505: sprite 'P', drapes "Q#*ltr" (Q plain,
                                curtain = the FULL cue in d_bits[0], halved on the device by which goal was
                                drawn; the other five Scrollys over static patterns, '*' per env in
                                d_pattern[2]).  Rewards are float64: pcl_outputs.d_reward_f64 is required.
                                program_arg = level, cue_after_teleport, timeout frames (PCL_T_MAZE_NO_TIMEOUT
                                = inf), teleport_delay, limbo_time.  Records: every Scrolly's AUX0 = its
                                np.roll offset (rows << 16 | cols); 't' AUX1 = teleport delay left, AUX2 =
                                limbo countdown; 'Q' AUX0 = which_goal (0 left, 1 right), AUX1 =
                                yo_we_have_teleported, AUX2 = the teleporter's in-limbo flag.  Plot AUX0 =
                                timeout_frames, AUX1 = teleportation_order_frame (-1 = unset), AUX2 / AUX3 =
                                teleportation_order.  d_rng, when bound, is u32 [B, 2, PCL_MT_WORDS]: slot 0
                                Python random.Random words (the cue), slot 1 NumPy RandomState words (the
                                speckle); d_pattern_init[2] then holds the UN-speckled '*' pattern */
  PCL_PROG_COMPILED = 14,    /* any registered MazeWalker / Scrolly / plain Drape classes: their update()
                                bodies compiled to the bytecode below (pcl_bind_code) and interpreted one
                                warp per env, in one scrolling group.  Registers: sprite AUX0-AUX2 (an
                                egocentric walker: AUX2 only; AUX0 / AUX1 hold its permits), a Scrolly's
                                AUX0-AUX2 (words 0-4 are its corners and last move frame), all eight
                                words of a plain drape record, plot AUX0-AUX3 (the_plot keys).
                                program_arg[2]: bit d set = Scrolly d writes its pattern (PCL_OP_SETPAT):
                                d_pattern[d] is then per env and reset from d_pattern_init[d] (per level),
                                and its curtain, the pattern window as of its last motion helper
                                (drapes.py:689-695), is kept in d_bits[d] (reset from d_bits_init[d]).
                                Other Scrolly patterns are static.  program_arg[3]: bit s set = sprite s
                                is a plain Sprite (things.py:265-391), not a MazeWalker: its code sets
                                its own position and visibility (PCL_OP_SETFIELD), its registers are
                                VROW, VCOL and AUX0-AUX2, and it may stand anywhere, off the board too.
                                Egocentric sprites may not set the bit.  program_arg[0] = 1: rewards are float64
                                (pcl_outputs.d_reward_f64 is required), 0: int32.  program_arg[1] =
                                the number of RNG slots the code draws from (0-2); with slots,
                                pcl_state.d_rng is required and is u32 [B, program_arg[1],
                                PCL_MT_WORDS], each slot the words of NumPy's RandomState or of
                                Python's random.Random, continued across auto-resets.  program_arg[4] = 1:
                                the game's Backdrop has compiled update() code (a function of its own,
                                header word 1 + n of the bytecode) that runs once per step before update
                                group 0 and writes a per-env live curtain, bound with pcl_bind_backdrop;
                                d_backdrop is then its per-level reset template (0: the backdrop is
                                static and d_backdrop is read directly) */
  PCL_PROG_BOX_WORLD = 15,   /* examples/research/box_world/box_world.py:127-271: sprite '.' (MazeWalker,
                                impassable '#', confined), NO drapes.  Every key 'a'-'t', lock 'A'-'T' and
                                the gem '*' is a cell of a per-env object grid held in d_bits[0] viewed as
                                u8 [rows, pitch] (bits_words = pitch / 4): 0 = no object, else the
                                character, bit 7 set on a distractor lock cell; d_bits_init[0] is the
                                level's reset template.  A held key sits at (0, 0).  rows <= 32 and
                                pitch <= 32 (grid_size <= 30).  program_arg[0] = max_num_steps.  Sprite
                                AUX0 = _step_counter; plot AUX0 = the character of the_plot['over_this']
                                (0 = unset), AUX1 = its position (row << 16 | col).  Rewards are int32
                                (the reference's floats 0, +1, -1, +10).  Levels have a '#' ring; without
                                it a look-up at row or column -1 wraps as NumPy's does, one past the last
                                row or column latches PCL_ENV_ERR_INDEX (NumPy's IndexError) and skips the
                                rest of the step's logic, and the walker never leaves the board.  pcl_layers and
                                pcl_export_curtain see the backdrop and the player only: object planes
                                are d_bits[0] == character */
  PCL_PROG_CUED_CATCH = 16,  /* examples/research/lp-rnn/cued_catch.py:96-317: sprites 'P' (MazeWalker, impassable '',
                                confined), 'a' and 'b' (plain Sprites: record VROW / VCOL = the start position),
                                drape 'Q' (curtain bit rows in d_bits[0]; d_bits_init[0] = the art's 'Q', which
                                stays in every row outside the bands 1:3, 3:5 and -2: that update() rewrites).
                                rows <= 32, cols <= 64.  Records: P AUX0 = _trials_till_reward; Q CORNER_R =
                                phase (0 first, 1 second), CORNER_C = first-phase tick, PRE_R = second-phase cue
                                choice, PRE_C = second-phase tick, LAST_FRAME = last reset frame (PCL_NEVER =
                                -inf), AUX0 = trials left, AUX1 = the cue->ball pairings (bit k set: cue k is
                                'top').  Plot AUX0 = programming_complete, AUX1 = which_ball (0 unset, 1 top,
                                2 bottom), AUX2 = last_ball_reset (PCL_NEVER = unset), AUX3 = 1 when this step's
                                reward is a Python float (the normalvariate branch), 0 for an int.
                                program_arg[0] = reward_sigma != 0: rewards are then float64
                                (pcl_outputs.d_reward_f64 is required), else int32; [1] =
                                initial_cue_duration (>= 1), [2] = cue_duration, [3] bit 0 =
                                always_show_ball_symbol, bit 1 = take the pairings from the template at a
                                start instead of drawing them (a facade whose Python CueDrape drew them);
                                [4] / [5] = reward_sigma as float64 bits (lo / hi), [6] / [7] = Lib/random.py's
                                NV_MAGICCONST as float64 bits (lo / hi).  d_rng is required: u32 [B,
                                PCL_MT_WORDS], the words of Python's random.Random, continued across steps and
                                auto-resets (random.sample at a start, randrange(4) per trial, normalvariate
                                per paid frame).  normalvariate's accept test zz <= -log(u2) uses the device's
                                double log (1 ulp) away from the boundary, and the correctly rounded
                                -log(u2) when zz lies within a few ulps of it */
  PCL_PROG_SEQUENCE_RECALL = 17, /* examples/research/lp-rnn/sequence_recall.py:107-317: sprite 'P' (MazeWalker,
                                impassable '#', confined), drapes 'M' (bit rows in d_bits[0], rewritten
                                whenever its record's AUX0, the set of covered lights '1'-'4' as bits 0-3,
                                changes) and '%' (art mask in d_bits_init[1], live rows in d_bits[1], record
                                AUX0 = cleared).  Backdrop characters are ' #1234' only.  rows <= 32,
                                cols <= 64.  Plot AUX0 = the program counter over _make_program's list (pc 2k
                                / 2k+1: OFF / ON of light k; 2L: the pause OFF; 2L+1+2k / 2L+2+2k: SEEK /
                                EXIT of light k; 4L: QUIT), AUX1 = frames_in_state, AUX2 = timeout_frames
                                (PCL_SEQUENCE_RECALL_NO_TIMEOUT = inf), AUX3 = the light sequence, light k in
                                bits 2k..2k+1 (0-3 for '1'-'4').  program_arg = sequence_length L (1-16),
                                demo_light_on_frames, demo_light_off_frames, max(1, pause_frames).  Rewards
                                are float64: pcl_outputs.d_reward_f64 is required.  With d_rng bound (u32 [B,
                                PCL_MT_WORDS], Python random.Random words) the sequence is redrawn at every
                                (re)start as L calls to random.choice('1234'), else taken from the template */
  PCL_PROG_ORDEAL = 8        /* examples/ordeal.py:74-266: program_arg[0] = PCL_ORDEAL_* chapter;
                                plot words AUX0 has_sword, AUX1 last_position (row << 16 | col,
                                -1 unset), AUX2 next_chapter chosen on the device, AUX3 prior chapter */
} pcl_program;

/* PCL_PROG_ORDEAL chapters (storytelling.Story keys of ordeal.py:94-97); AUX2 holds
 * PCL_ORDEAL_NEXT_UNSET until an entity names the next chapter, PCL_ORDEAL_NEXT_NONE for
 * `next_chapter = None`. */
enum { PCL_ORDEAL_NEXT_UNSET = -1, PCL_ORDEAL_NEXT_NONE = 0,
       PCL_ORDEAL_CASTLE = 1, PCL_ORDEAL_CAVERN = 2, PCL_ORDEAL_KANSAS = 3 };

/* PCL_PROG_T_MAZE: program_arg[2] for timeout_frames = -1 (never times out). */
#define PCL_T_MAZE_NO_TIMEOUT 0x7fffffff

/* PCL_PROG_SEQUENCE_RECALL: plot AUX2 for timeout_frames = inf (never times out). */
#define PCL_SEQUENCE_RECALL_NO_TIMEOUT 0x7fffffff

/* PCL_PROG_CLASSICS: pcl_spec.program_arg[0] selects the rule set; the games
 * pay float rewards (1.0, -1.0, -100.0, 100.0) which d_reward carries as the
 * equal int32 value. */
enum { PCL_CLASSIC_FOUR_ROOMS = 0, /* four_rooms.py:52-80; program_arg[1..2] = goal cell (4, 3) */
       PCL_CLASSIC_CLIFF_WALK = 1, /* cliff_walk.py:46-86 */
       PCL_CLASSIC_CHAIN_WALK = 2, /* chain_walk.py:44-73 */
       PCL_CLASSIC_FLUVIAL = 3     /* examples/fluvial_natation.py:61-110 (int rewards); program_arg[1..2] =
                                      first / end row of the flowing backdrop band (1, 4); the
                                      rotation count is plot word PCL_P_AUX0 */ };

/* Plot directives as action words of PCL_PROG_FIXTURE (plot.py:136-260). */
#define PCL_FIXTURE_DIRECTIVES 4
enum { PCL_DIR_NONE = 0,
       PCL_DIR_ADD_REWARD = 1,        /* arg = int32 reward (plot.py:201-214) */
       PCL_DIR_TERMINATE = 2,         /* arg = f32 bits of the discount in [0, 1] (plot.py:176-199) */
       PCL_DIR_DEFAULT_DISCOUNT = 3,  /* arg = f32 bits (plot.py:247-260; upstream resets the default
                                         to 1.0 after every step, plot.py:345-356) */
       PCL_DIR_Z_ORDER = 4 };         /* arg = move_this | in_front_of << 8, 0 = None (plot.py:136-174) */

/* PCL_PROG_COMPILED bytecode (pcl_bind_code): int32 words.  Word 0 = n, the number of entities
 * (n_sprites + n_drapes); words 1..n = the first word of each entity's update() (sprites first,
 * then drapes, in spec order); with program_arg[4] set, word 1 + n = the first word of the
 * Backdrop's update().  Entities of one class share their code.  The entry points split
 * the words after the header into functions; each ends with PCL_OP_RET, and its jumps go
 * forward to a word inside it, so every update ends.  The operand stack holds int32 values;
 * "pop r, c" pops c first.  An entity operand of -1 means the entity being updated.  Cell
 * indices follow NumPy: a negative index counts from the end once, anything else off the board
 * latches PCL_ENV_ERR_INDEX and reads 0 / writes nothing.  Integers wrap at 32 bits. */
#define PCL_MAX_CODE_WORDS 16384
#define PCL_CODE_STACK 16    /* operand stack slots per update */
#define PCL_CODE_LOCALS 16   /* local variable slots per update */
enum {
  PCL_OP_RET = 0,       /* end of this entity's update                                       */
  PCL_OP_PUSH,          /* imm: push imm                                                      */
  PCL_OP_POP,           /* pop                                                                */
  PCL_OP_DUP,           /* push a copy of the top                                             */
  PCL_OP_LOAD,          /* slot: push local `slot`                                            */
  PCL_OP_STORE,         /* slot: pop into local `slot`                                        */
  PCL_OP_JMP,           /* target: jump (target > this word)                                  */
  PCL_OP_JZ,            /* target: pop; jump if it is 0                                       */
  PCL_OP_JNZ,           /* target: pop; jump if it is not 0                                   */
  PCL_OP_ADD, PCL_OP_SUB, PCL_OP_MUL,
  PCL_OP_FLOORDIV,      /* Python `//` and `%`: floor semantics; by zero latches PCL_ENV_ERR_ARITH */
  PCL_OP_MOD,
  PCL_OP_EQ, PCL_OP_NE, PCL_OP_LT, PCL_OP_LE, PCL_OP_GT, PCL_OP_GE,   /* pop b, a; push a op b */
  PCL_OP_NEG, PCL_OP_NOT,
  PCL_OP_EQ2,           /* pop (r2, c2), (r1, c1); push r1 == r2 && c1 == c2                  */
  PCL_OP_IN,            /* k, v_1 .. v_k: pop x; push whether x is one of the v_i (k <= 64)     */
  PCL_OP_ACTION,        /* push the env's action (PCL_ACTION_NONE at a (re)start)            */
  PCL_OP_FRAME,         /* push the_plot.frame                                                */
  PCL_OP_FIELD,         /* sprite, f: push row, col, virtual row, virtual col, visible (f 0-4) */
  PCL_OP_GETR,          /* k: push register k of the entity being updated (walker k < 3, plain
                           sprite k < 5)                                                       */
  PCL_OP_SETR,          /* k: pop into it                                                     */
  PCL_OP_GETP,          /* k: push plot register k (k < 4)                                    */
  PCL_OP_SETP,          /* k: pop into it                                                     */
  PCL_OP_BOARD,         /* pop r, c; push the board of the last render at (r, c)             */
  PCL_OP_BACKDROP,      /* pop r, c; push the backdrop at (r, c)                              */
  PCL_OP_CURTAIN,       /* drape: pop r, c; push its curtain at (r, c)                        */
  PCL_OP_SETCELL,       /* pop r, c, v; the updated drape's curtain at (r, c) = v != 0        */
  PCL_OP_FILL,          /* pop v; every cell of the updated drape's curtain = v != 0          */
  PCL_OP_ANY,           /* drape: push whether its curtain has a cell set                     */
  PCL_OP_MOVE,          /* motion (PCL_M_N .. PCL_M_STAY): move the updated walker; push 1 if
                           it was blocked, 0 if it moved (upstream: None)                     */
  PCL_OP_TELEPORT,      /* pop r, c: the updated walker's _teleport((r, c))                   */
  PCL_OP_REWARD,        /* pop x: the_plot.add_reward(x)                                      */
  PCL_OP_REWARD_F64,    /* lo, hi: add_reward of the float64 with these bit halves            */
  PCL_OP_TERMINATE,     /* f32 bits: the_plot.terminate_episode(discount)                     */
  PCL_OP_DISCOUNT,      /* f32 bits: the_plot.change_default_discount(discount)              */
  /* Draws from the env's RNG slot `slot` of pcl_state.d_rng (slot < program_arg[1]). */
  PCL_OP_RANDINT,       /* slot, rule (PCL_RAND_*): pop low, high; push a draw from the rule's
                           range.  An empty range latches PCL_ENV_ERR_RANGE, pushes low and
                           consumes no output                                                  */
  PCL_OP_RANDCMP,       /* slot, cmp, lo, hi: draw a float (two outputs, 53 bits, as NumPy's
                           random_sample() and Python's random()) and push `draw cmp x`, x the
                           float64 with bit halves lo / hi, cmp 0-5 = == != < <= > >=          */
  PCL_OP_PICK,          /* k, v_1 .. v_k: pop i; push v_(i+1) (1 <= k <= 64); i outside 0 .. k-1
                           latches PCL_ENV_ERR_INDEX and pushes 0                              */
  /* Scrollys (drapes.py:378-695).  `scrolly` operands name a Scrolly drape, -1 only inside a
   * Scrolly's own update.  CURTAIN and ANY on a Scrolly read its curtain. */
  PCL_OP_SCROLL,        /* motion: _maybe_move of the updated Scrolly (drapes.py:487-659)       */
  PCL_OP_PRESCROLL,     /* scrolly: pop r, c; refresh its pre-scroll corner if it has not moved
                           in this frame (drapes.py:407-408); push (r + pre_r, c + pre_c)      */
  PCL_OP_POSTSCROLL,    /* scrolly: pop r, c; push (r + corner_r, c + corner_c); if it has not
                           moved in this frame, latch PCL_ENV_ERR_POSTSCROLL                   */
  PCL_OP_PATTERN,       /* scrolly: pop r, c; push its whole_pattern at (r, c) (NumPy indexing
                           over pattern_rows x pattern_cols)                                  */
  PCL_OP_SETPAT,        /* pop r, c, v: the updated Scrolly's whole_pattern at (r, c) = v != 0
                           (its program_arg[2] bit must be set)                                */
  PCL_OP_PATANY,        /* scrolly: push whether its whole_pattern has a cell set             */
  /* Plain Sprites (program_arg[3]).  Their positions are any int32 pair.  A render paints a
   * visible one at its NumPy-wrapped cell; one still off the board after the wrap latches
   * PCL_ENV_ERR_INDEX at the render that follows its update group and paints nothing
   * (rendering.py:139, `board[tuple(position)]`). */
  PCL_OP_SETFIELD,      /* f: pop v into the updated plain sprite's row (f 0), col (f 1) or
                           visible bit (f 4, v != 0); the write twin of FIELD                 */
  /* The Backdrop's update() (program_arg[4]): these three appear only in its function, which
   * has no registers, no motion, no drape or pattern writes and no -1 entity operand.  They
   * write the env's live curtain; BACKDROP reads it, and every later render paints it. */
  PCL_OP_SETBACK,       /* pop r, c, v: the live curtain at (r, c) = v (as a byte)             */
  PCL_OP_FILLBACK,      /* pop v: every cell of the live curtain = v (as a byte)              */
  PCL_OP_ROLLBACK,      /* axis, lo, hi: pop shift; rows lo .. hi - 1 = np.roll(those rows, shift,
                           axis) (axis 0 or 1, 0 <= lo <= hi <= rows)                         */
  PCL_OP_COUNT
};

/* PCL_OP_RANDINT rules, over int32 operands with widths computed in 64 bits:
 *   PCL_RAND_NUMPY        RandomState.randint(low, high): [low, high); one 32-bit output per
 *                         try, masked rejection; no output when the range holds one value;
 *   PCL_RAND_PYTHON       Random.randrange(low, high): low + _randbelow(high - low), where
 *                         _randbelow(n) repeats getrandbits(n.bit_length()) until it is < n
 *                         (getrandbits(k <= 32) = one output >> (32 - k); k == 33 = two
 *                         outputs lo, hi: lo | (hi >> 31) << 32), so a width of 1 consumes output;
 *   PCL_RAND_PYTHON_CLOSED Random.randint(low, high): as PCL_RAND_PYTHON over [low, high]. */
enum { PCL_RAND_NUMPY = 0, PCL_RAND_PYTHON = 1, PCL_RAND_PYTHON_CLOSED = 2 };

/* Motion codes (prefab_parts/sprites.py:140-150). */
enum { PCL_M_N = 0, PCL_M_NE, PCL_M_E, PCL_M_SE, PCL_M_S, PCL_M_SW, PCL_M_W,
       PCL_M_NW, PCL_M_STAY, PCL_M_NONE = -1 };

/* Action value meaning "actions=None" (the its_showtime() frame,
 * engine.py:581). */
#define PCL_ACTION_NONE (-1)

/* Sprite record layout, int32[PCL_SPRITE_WORDS] (things.py:339-391,
 * sprites.py:153-205). */
enum { PCL_S_ROW = 0, PCL_S_COL, PCL_S_VROW, PCL_S_VCOL,
       PCL_S_FLAGS,          /* bit0 visible; bits1-2 prior_visible: 0 None, 1 False, 2 True */
       PCL_S_AUX0,           /* program-specific (e.g. patroller heading; permit mask)      */
       PCL_S_AUX1,           /* program-specific (e.g. permit frame)                        */
       PCL_S_AUX2 };
/* Drape record layout, int32[PCL_DRAPE_WORDS] (drapes.py:293-376). */
enum { PCL_D_CORNER_R = 0, PCL_D_CORNER_C, PCL_D_PRE_R, PCL_D_PRE_C,
       PCL_D_LAST_FRAME,     /* _last_maybe_move_frame; INT32_MIN = -inf */
       PCL_D_AUX0, PCL_D_AUX1, PCL_D_AUX2 };
/* Plot record layout, int32[PCL_PLOT_WORDS] (plot.py:69-104,
 * protocols/scrolling.py:198-241). */
enum { PCL_P_FRAME = 0, PCL_P_GAME_OVER, PCL_P_ERROR, PCL_P_EPISODES,
       PCL_P_ORDER_R, PCL_P_ORDER_C, PCL_P_ORDER_FRAME, PCL_P_EGO_MASK,
       PCL_P_AUX0, PCL_P_AUX1, PCL_P_AUX2, PCL_P_AUX3,
       PCL_P_CROP_R, PCL_P_CROP_C, PCL_P_CROP_INIT, PCL_P_RESERVED };

/* Scrolling-group record layout, int32[PCL_GROUP_WORDS]: the per-group part of the
 * blackboard of protocols/scrolling.py:198-241.  Group 0 lives in the plot record
 * (PCL_P_ORDER_R .. PCL_P_EGO_MASK); groups 1.. in pcl_state.d_groups. */
enum { PCL_G_ORDER_R = 0, PCL_G_ORDER_C, PCL_G_ORDER_FRAME, PCL_G_EGO_MASK };

/* Static description of one game (what Engine's set-up API collected:
 * engine.py:248-518).  All envs of a handle share it. */
typedef struct pcl_spec {
  int32_t abi_version;           /* PCL_ABI_VERSION */
  int32_t program;               /* pcl_program */
  int32_t rows, cols;            /* board H x W (engine.py:202-203) */
  int32_t pitch;                 /* bytes per board row in HBM, multiple of 16, >= cols */
  int32_t n_sprites, n_drapes;
  int32_t auto_reset;            /* 1: an env that is game-over is rebuilt by the next step */
  int32_t pattern_rows, pattern_cols; /* Scrolly whole_pattern shape (drapes.py:338-343) */
  int32_t pattern_words;         /* uint32 words per bit-packed pattern row, even and zero padded.
                                    PCL_PROG_SCROLLY_MAZE needs >= ceil(pattern_cols/32) + 1 and
                                    >= ((pattern_cols - cols) / 32 rounded down to even) + nw, where
                                    nw = 2 * ceil((63 + cols) / 64) words, at least 4, are staged per
                                    window row */
  int32_t bits_words;            /* uint32 words per bit-packed board-sized row */
  uint8_t sprite_char[PCL_MAX_SPRITES];
  uint8_t drape_char[PCL_MAX_DRAPES];
  uint32_t impassable[PCL_MAX_SPRITES][4]; /* 128-bit ASCII set (sprites.py:190) */
  int32_t sprite_confined[PCL_MAX_SPRITES];
  int32_t sprite_egocentric[PCL_MAX_SPRITES];
  int32_t margins[PCL_MAX_DRAPES][2];      /* Scrolly scroll_margins; -1,-1 = None */
  uint8_t z_order[PCL_MAX_SPRITES + PCL_MAX_DRAPES]; /* initial z-order, chars */
  int32_t n_groups;
  int32_t group_len[PCL_MAX_SPRITES + PCL_MAX_DRAPES];
  uint8_t group_chars[PCL_MAX_SPRITES + PCL_MAX_DRAPES]; /* update order, concatenated */
  int32_t drape_kind[PCL_MAX_DRAPES];      /* 0 = plain bool curtain (d_bits), 1 = Scrolly (d_pattern) */
  int32_t program_arg[8];                  /* per-program constants (see pcl_program); else 0 */
  /* Scrolling groups (`scrolling_group` of MazeWalker / Scrolly, sprites.py:176,
   * drapes.py:309): index of each entity's group, 0 .. n_scroll_groups - 1.  Only
   * PCL_PROG_FIXTURE accepts more than one group; 0 groups means 1. */
  int32_t n_scroll_groups;
  int32_t sprite_group[PCL_MAX_SPRITES];
  int32_t drape_group[PCL_MAX_DRAPES];
} pcl_spec;

/* Device buffers of one handle (all caller-owned).  A "*_bstride" is the
 * distance between consecutive envs in ELEMENTS of that array; 0 means all
 * envs share one copy (legal only for arrays the step never writes). */
typedef struct pcl_state {
  /* static level data */
  const uint8_t* d_backdrop;   int64_t backdrop_bstride;       /* u8 [*, rows, pitch] */
  /* Scrolly patterns, bit-packed: u32 [*, pattern_rows, pattern_words], cell c
   * of a row is bit (c & 31) of word (c >> 5). */
  uint32_t* d_pattern[PCL_MAX_DRAPES];  int64_t pattern_bstride[PCL_MAX_DRAPES];
  const uint32_t* d_pattern_init[PCL_MAX_DRAPES]; int64_t pattern_init_bstride[PCL_MAX_DRAPES];
  /* board-sized bit-packed curtains for non-Scrolly drapes: u32 [*, rows, bits_words] */
  uint32_t* d_bits[PCL_MAX_DRAPES];     int64_t bits_bstride[PCL_MAX_DRAPES];
  const uint32_t* d_bits_init[PCL_MAX_DRAPES]; int64_t bits_init_bstride[PCL_MAX_DRAPES];
  /* per-env registers and their reset templates */
  int32_t* d_sprites;  const int32_t* d_sprites_init; int64_t sprites_init_bstride; /* [B, S, 8] */
  int32_t* d_drapes;   const int32_t* d_drapes_init;  int64_t drapes_init_bstride;  /* [B, D, 8] */
  int32_t* d_plot;     const int32_t* d_plot_init;    int64_t plot_init_bstride;    /* [B, 16]   */
  uint32_t* d_rng;     /* MT19937 per env, u32 [B, PCL_MT_WORDS]; NULL if unused.  PCL_PROG_T_MAZE
                          and PCL_PROG_COMPILED keep several slots per env: u32 [B, slots,
                          PCL_MT_WORDS] (see their pcl_program entries) */
  /* per-env z-order (chars, back to front) for programs whose entities issue
   * Plot.change_z_order (engine.py:796-835): u8 [B, n_sprites + n_drapes]; NULL = spec z_order */
  uint8_t* d_z_order;  const uint8_t* d_z_order_init; int64_t z_order_init_bstride;
  /* Scrolling groups 1 .. n_scroll_groups - 1 (group 0 is in the plot record):
   * i32 [B, PCL_MAX_SCROLL_GROUPS, PCL_GROUP_WORDS], slot 0 unused; NULL when the
   * game has a single group. */
  int32_t* d_groups;   const int32_t* d_groups_init;  int64_t groups_init_bstride;
  /* Level sharing: envs that play the same level need only one copy of its
   * static data.  When d_level (i32 [B]) is non-NULL, every array the step never
   * writes — d_backdrop, read-only patterns, every *_init template — is indexed
   * by d_level[env] instead of env (the *_bstride is then the per-LEVEL stride);
   * mutable arrays stay env-indexed.  NULL = env-indexed (or bstride 0). */
  const int32_t* d_level;
} pcl_state;

/* Per-step outputs = the (observation, reward, discount) triple of
 * Engine.play() (engine.py:639) plus Engine.game_over (engine.py:657). */
typedef struct pcl_outputs {
  uint8_t* d_board;       /* u8 [B, rows, pitch]; Observation.board.  PCL_PROG_FIXTURE reads the
                             board of the LAST render back from here at the next step (its
                             entities may test any character, engine.py:725-735): pass the same
                             d_board to consecutive steps of a handle running that program.
                             PCL_PROG_SCROLLY_MAZE repaints only the cells that can have changed
                             when d_board holds the env's last render (the buffer of the handle's
                             previous step or reset) and neither window scrolls: a host that writes
                             into a step's board buffer passes a different buffer to the next step
                             or reset, or calls pcl_bind_state again, which paints every board. */
  int32_t* d_reward;      /* i32 [B]; summed reward (plot.py:201-214), 0 if none */
  uint8_t* d_has_reward;  /* u8 [B]; 0 = reference returned reward None */
  float*   d_discount;    /* f32 [B]; 1.0 running / 0.0 terminated unless a directive said otherwise
                             (plot.py:104,176-199,247-260) */
  uint8_t* d_done;        /* u8 [B]; Engine.game_over after this step: 0 running, 1 ended by the
                             game, PCL_DONE_TIME_LIMIT ended by the time limit (pcl_set_time_limit) */
  double*  d_reward_f64;  /* f64 [B]; the summed reward exactly as the reference's float sum produces
                             it, 0.0 if none.  Written only by programs whose rewards are not integers
                             (PCL_PROG_T_MAZE and PCL_PROG_SEQUENCE_RECALL always, PCL_PROG_COMPILED
                             and PCL_PROG_CUED_CATCH when program_arg[0] is set), which then leave
                             d_reward alone; required by them (PCL_ERR_INVALID when NULL), ignored by
                             every other program. */
} pcl_outputs;

typedef struct pcl_handle pcl_handle;

/* Validate `spec`, allocate the handle.  Replaces Engine.__init__ + set-up
 * bookkeeping (engine.py:191-246). */
int pcl_create(const pcl_spec* spec, int batch, int device, pcl_handle** out);
int pcl_destroy(pcl_handle* h);

/* Attach the caller's device buffers.  The static level data (backdrop, read-only
 * patterns, reset templates) may be read into the handle's own derived copies before
 * the first step or reset after this call; a host that rewrites it afterwards calls
 * pcl_bind_state again. */
int pcl_bind_state(pcl_handle* h, const pcl_state* state);

/* PCL_PROG_COMPILED: the bytecode every env runs, h_code a HOST array of n_words int32 words
 * (see PCL_OP_*).  It is checked before anything touches a device: known opcodes, entry
 * points that split the code into functions of the right entity kind, each ending in
 * PCL_OP_RET, forward jumps inside the function, entity, register, local and stack bounds,
 * n_words <= PCL_MAX_CODE_WORDS; PCL_ERR_INVALID otherwise.  The handle keeps a copy; the
 * next pcl_reset / pcl_step / pcl_run / pcl_run_many / pcl_step_host* of the handle uploads
 * it on its own stream and waits for that copy before it launches (it synchronises that
 * stream once, so that call must not be captured into a CUDA graph), after which launches on
 * any stream read the new code.  Binding again while kernels of the handle still run is
 * safe: the upload first waits for the device.  Other programs: PCL_ERR_UNSUPPORTED.
 * pcl_reset / pcl_step return PCL_ERR_UNBOUND until code is bound. */
int pcl_bind_code(pcl_handle* h, const int32_t* h_code, int32_t n_words);

/* PCL_PROG_COMPILED with program_arg[4] set: the Backdrop's live curtains, u8 [B, rows, pitch]
 * (caller-owned DEVICE memory).  A (re)start copies the env's level template (d_backdrop,
 * indexed through d_level) into its row; the Backdrop's code then writes it, the step's renders
 * and pcl_layers read it.  PCL_ERR_INVALID for a NULL buffer and for every other handle.  The
 * step and reset entry points of such a handle return PCL_ERR_UNBOUND until it is bound. */
int pcl_bind_backdrop(pcl_handle* h, uint8_t* d_backdrop_live);

/* Engine.its_showtime() (engine.py:520-581) for every env whose d_env_mask
 * byte is non-zero (NULL = all): restore the reset templates, then run the
 * actions=None frame.  Envs not selected are left untouched. */
int pcl_reset(pcl_handle* h, const uint8_t* d_env_mask, const pcl_outputs* out,
              void* stream);

/* Engine.play(actions) (engine.py:583-639) for all envs in lockstep: one fused
 * kernel = _update_and_render + _apply_and_clear_plot.  d_actions is
 * i32 [B, actions_per_env]: actions_per_env = 1 for the example games;
 * PCL_PROG_FIXTURE takes n_sprites + n_drapes + 2 * PCL_FIXTURE_DIRECTIVES words per
 * env: one motion code per entity in update order, then PCL_FIXTURE_DIRECTIVES
 * (opcode, argument) pairs — the Plot directives the entities issued this step, in
 * call order (the last discount-setting call wins, as upstream). */
int pcl_step(pcl_handle* h, const int32_t* d_actions, const pcl_outputs* out,
             void* stream);

/* T consecutive pcl_step()s with d_actions i32 [T, B, actions_per_env]; the
 * outputs hold the last step's values. */
int pcl_run(pcl_handle* h, const int32_t* d_actions, int steps,
            const pcl_outputs* out, void* stream);

/* A rollout (pcl_rollout): what each of T steps produced, kept in caller-owned [T, B, ...]
 * buffers.  Every d_* field is a DEVICE pointer and NULL means "not kept"; the spec
 * pointers are HOST pointers read during the call.  Slot t of a [T, B, ...] buffer starts
 * t * B * (elements per env) elements from its base.
 *   Per-step outputs, as pcl_outputs after step t: d_reward i32 [T, B] (int-reward
 *   programs) or d_reward_f64 f64 [T, B] (float-reward programs; the other one is ignored),
 *   d_has_reward u8 [T, B], d_discount f32 [T, B], d_done u8 [T, B].
 *   d_attached: the attached cropper's view after every step, u8 [T, B, crop rows, crop
 *   cols].  The attached cropper is the handle's own (pcl_attach_cropper, run inside the
 *   step kernel) or, for programs without that epilogue, `crop` below.
 *   crop, d_crop_state, d_crop: a cropper run after every step (pcl_crop(crop, board,
 *   d_crop, d_crop_state)), for handles with no cropper attached; its view goes to
 *   slot t of d_attached when that is kept, else to d_crop (u8 [B, crop rows, crop cols]).
 *   observe, ...: one post-processor after every step, NULL = none.  With observe_crop
 *   NULL it is pcl_observe over the board; with it, pcl_crop_observe over that window
 *   (its corner in d_observe_state).  d_view is the base of slot 0, view_stride_t the
 *   ELEMENTS between slots, and observe's strides address one slot.  Over the board a
 *   depth past 32 is split into launches of at most 32 planes, and d_table then holds the
 *   tables of those launches one after another, [128, n] each (for depth <= 32 that is
 *   [128, depth]); over a window d_table is [128, depth].  d_unknown (i32 [1], may be
 *   NULL) is set to 1 when any step's view met an unknown character. */
struct pcl_crop_spec;
struct pcl_observe_spec;
typedef struct pcl_rollout_rec {
  int32_t* d_reward;
  double* d_reward_f64;
  uint8_t* d_has_reward;
  float* d_discount;
  uint8_t* d_done;
  uint8_t* d_attached;
  const struct pcl_crop_spec* crop;
  int32_t* d_crop_state;
  uint8_t* d_crop;
  const struct pcl_observe_spec* observe;
  const struct pcl_crop_spec* observe_crop;
  int32_t* d_observe_state;
  const void* d_table;
  const uint8_t* d_valid;
  int32_t* d_unknown;
  void* d_view;
  int64_t view_stride_t;
} pcl_rollout_rec;

/* T = `steps` steps from one call: step t is pcl_step(h, d_actions + t * B *
 * actions_per_env, out), then the attached cropper, then rec's observer: the launches
 * pcl_step, pcl_crop and pcl_observe / pcl_crop_observe would make, in that order, with
 * what they wrote sent to slot t of rec's buffers.  rec == NULL keeps nothing: that is
 * pcl_run.  The board stays out->d_board at every step (boards are not kept: an identity
 * repaint as the observer keeps them).  Afterwards `out` and the attached cropper's view
 * hold step T-1's values, as after T pcl_step calls.
 * Without auto_reset, an env frozen at step t (game over before it) writes nothing in that
 * step; its slots of the kept outputs then hold done 1, has_reward 0, reward 0 and discount
 * 0.0, and its view slots the view of its unchanged board.  (When the outputs are kept,
 * `out` of an env frozen at step T-1 holds that record too.)
 * Everything is checked once, with the statuses of the single entry points (a tracking list
 * naming a drape is PCL_ERR_UNSUPPORTED: no curtains are exported between steps); then the
 * launches are enqueued with no allocation and no host synchronisation, so the call can be
 * captured into a CUDA graph.  Consecutive step launches are block-chained as pcl_run's
 * are when no other kernel lies between them (no observer, no cropper after the step).
 * pcl_rollout_episodes (below) also keeps each step's episode return and length. */
int pcl_rollout(pcl_handle* h, const int32_t* d_actions, int steps, const pcl_outputs* out,
                const pcl_rollout_rec* rec, void* stream);
/* sizeof(pcl_rollout_rec), for bindings to verify their layout at load time. */
int pcl_rollout_rec_size(void);

/* `steps` pcl_step()s issued from one C call over several handles in rotation:
 * step t advances handles[t % n_handles] with d_actions[t] (HOST array of `steps`
 * device pointers, each i32 [B, actions_per_env] of that handle) into
 * outs[t % n_handles].  The batched stand-in for a driver looping over many
 * Engines (one reference Engine per env, engine.py:583); nothing but kernel
 * launches sits between the steps, so the sequence can also be captured into a
 * CUDA graph on `stream`. */
int pcl_run_many(pcl_handle* const* handles, int n_handles, const int32_t* const* d_actions,
                 const pcl_outputs* const* outs, int steps, void* stream);

/* Episode time limit.  pcl_set_time_limit(h, L) with L >= 1: a step that leaves an env at
 * frame L or later ends its episode, unless the game ended it in that same step.  An env's
 * frame is 0 after its its_showtime() frame (pcl_reset, or a restart under auto_reset) and
 * goes up by one per step, so with the limit set from the start the L-th step after a
 * (re)start is the last one.  Such a step reports done = PCL_DONE_TIME_LIMIT, and its plot
 * record's game-over word holds the same value; a game's own ending (terminate_episode,
 * including a game's own step limit such as box_world's max_num_steps) stays done 1.  A
 * truncated step's reward, has_reward, discount and board are what the step produced
 * without a limit: the discount is the game's (1.0 unless a directive changed it), which is
 * what value bootstrapping across a time limit wants.  The next step treats the env as after
 * any ending: a restart under auto_reset (action ignored, templates restored, episode count
 * + 1, random streams continued), else the env stays frozen and a rollout's slots hold the
 * frozen record (done 1).  A masked pcl_reset starts an env's count afresh, which is how a
 * host staggers its envs' episodes.
 * L = 0 (the default) is no limit: every output, record and kernel behaves as without this
 * call.  The limit is read when a step is launched: the next pcl_step, pcl_run, pcl_rollout,
 * pcl_run_many and pcl_step_host* of the handle use it, and a CUDA graph captured earlier
 * keeps the limit it was captured with.  PCL_ERR_INVALID for a NULL handle or L < 0.
 * Cost (DESIGN.md section 5; H100 80GB HBM3, 700 W): with the limit off bench.py's C2 step is
 * 6.33-6.39 us against the parent's 6.37; a wave of restarts the limit causes on C2 adds about
 * 7.5 us once per L + 1 steps. */
#define PCL_DONE_TIME_LIMIT 2
int pcl_set_time_limit(pcl_handle* h, int32_t max_frames);

/* Episode returns.  pcl_bind_episodes(h, d_return) binds a caller-owned f64 [B] device
 * buffer of running returns; NULL turns tracking off (the default).  With it bound, every
 * launch that steps or (re)starts an env updates that env's episode return R:
 *   r = the step's reward as a double: (double)reward for int32-reward programs (exact),
 *       the value stored to d_reward_f64 for float-reward programs, 0.0 when has_reward
 *       is 0;
 *   R = r when the step's frame is 0 (its_showtime: pcl_reset, or a restart under
 *       auto_reset), else R = R + r, one IEEE double addition per step in step order.
 * That is what `ret = r if frame == 0 else ret + r` computes in Python over the engine's
 * own outputs and plot frames.  The episode length is the plot's frame after the step (the
 * number of steps since the env's (re)start), so it is not stored again.  At a step with
 * done != 0, R and the frame are the finished episode's return and length; a truncated
 * episode's (PCL_DONE_TIME_LIMIT) return is the sum up to the cut.  An env a launch skips
 * writes nothing: a frozen env without auto_reset, an env a masked pcl_reset leaves alone.
 * R starts as whatever the buffer holds; the env's first (re)start after binding
 * overwrites it.
 * The binding is read when a step or reset is launched: pcl_step, pcl_reset, pcl_run,
 * pcl_run_many, pcl_rollout* and pcl_step_host* of the handle use it, and a CUDA graph
 * captured earlier keeps the binding it was captured with.  It survives pcl_bind_state.
 * Every output, record and board is the same with and without it; the work per env-step is
 * one 8-byte load and one 8-byte store, plus the kept slots in a rollout (DESIGN.md section 5
 * has what was measured).  PCL_ERR_INVALID for a NULL handle or a d_return that is not 8-byte
 * aligned. */
int pcl_bind_episodes(pcl_handle* h, double* d_return);

/* What pcl_rollout_episodes keeps of each step's episode, in caller-owned [T, B] DEVICE
 * buffers; NULL = not kept.  d_return f64 [T, B]: R after step t.  d_length i32 [T, B]:
 * the env's plot frame after step t. */
typedef struct pcl_episode_rec {
  double* d_return;
  int32_t* d_length;
} pcl_episode_rec;

/* pcl_rollout that also keeps every step's episode return and length (pcl_episode_rec);
 * ep == NULL is pcl_rollout.  A kept array needs a handle with bound returns
 * (pcl_bind_episodes) and an aligned pointer, else PCL_ERR_INVALID.  Without auto_reset the
 * kept slots of an env frozen at step t hold 0.0 and 0.  Afterwards the bound [B] buffer
 * holds R after step T-1, as after T pcl_step calls.  Launch and chaining counts are
 * pcl_rollout's. */
int pcl_rollout_episodes(pcl_handle* h, const int32_t* d_actions, int steps,
                         const pcl_outputs* out, const pcl_rollout_rec* rec,
                         const pcl_episode_rec* ep, void* stream);
/* sizeof(pcl_episode_rec), for bindings to verify their layout at load time. */
int pcl_episode_rec_size(void);

/* Seeded generators.  pcl_seed_rng writes, for every env whose d_env_mask byte is non-zero
 * (NULL = all), each of its n_slots generator slots in pcl_state.d_rng (u32 [B, n_slots,
 * PCL_MT_WORDS]) as a fresh generator seeded with d_seeds[env] (u32 [B], DEVICE) would hold
 * them.  h_kinds (HOST, n_slots values, in d_rng slot order) names each slot's rule.  For a
 * seed s in [0, 2^32):
 *   PCL_SEED_NUMPY   the words of np.random.RandomState(s) (NumPy's legacy seeding): key
 *                    word 0 is s, word i is 1812433253 * (w ^ (w >> 30)) + i of the word w
 *                    before it, and the position is 624;
 *   PCL_SEED_PYTHON  the words of random.Random(s).getstate()[1] (CPython's init_by_array
 *                    over the one-word key [s]): the key words of init_genrand(19650218),
 *                    the same for every seed, then its two mixing loops, then word 0 =
 *                    0x80000000, and the position is 624.
 * Either way the next draw twists first, as it does from any host-seeded words.  Unselected
 * envs, and every array but d_rng, are left untouched.  The call allocates nothing and does
 * not synchronise, so it can be captured into a CUDA graph.  The generators are all a restart
 * draws from, so a pcl_reset of the same mask after this call runs each env's its_showtime()
 * frame from its new words: that is Gymnasium's reset(seed=...), per env.  Draws made when
 * the game was built (the reset templates) are not redrawn.
 * Refusals, in order: PCL_ERR_INVALID for a NULL handle or NULL d_seeds; PCL_ERR_UNBOUND
 * before pcl_bind_state; PCL_ERR_UNSUPPORTED for a program with no generator slots;
 * PCL_ERR_INVALID when the bound d_rng is NULL, n_slots is not the program's slot count
 * (1 for PCL_PROG_MARAUDERS, _SHOCKWAVE, _APPREHEND, _CUED_CATCH and _SEQUENCE_RECALL, 2 for
 * PCL_PROG_T_MAZE, program_arg[1] for PCL_PROG_COMPILED), or h_kinds is NULL or holds a
 * value that is not a PCL_SEED_*.
 * Cost (DESIGN.md section 5; H100 80GB HBM3, 700 W): 54 us for 4096 envs of two slots, 420 us
 * for 65 536. */
enum { PCL_SEED_NUMPY = 0, PCL_SEED_PYTHON = 1 };
int pcl_seed_rng(pcl_handle* h, const uint8_t* d_env_mask, const uint32_t* d_seeds,
                 const int32_t* h_kinds, int n_slots, void* stream);

/* The host-buffer and hand-off entry points below (pcl_step_host, pcl_step_host_async,
 * pcl_pack_handoff, pcl_pack_handoff_peers, pcl_crop_handoff) carry an int32 reward in their
 * host buffers and records: they return PCL_ERR_UNSUPPORTED for a program with float64
 * rewards (PCL_PROG_T_MAZE).  Step those with pcl_step and read d_reward_f64. */

/* Host-buffer form of pcl_step: copies h_actions to the device, steps, copies
 * the outputs back into the h_* buffers (any may be NULL = skip) and
 * synchronises the stream.  `out` names the device staging buffers. */
int pcl_step_host(pcl_handle* h, const int32_t* h_actions, int32_t* d_actions,
                  const pcl_outputs* out, uint8_t* h_board, int32_t* h_reward,
                  uint8_t* h_has_reward, float* h_discount, uint8_t* h_done,
                  void* stream);

/* Pipelined form of pcl_step_host.  Enqueues H2D(actions) and the step on
 * `stream`, then the D2H of the requested outputs on a handle-owned copy stream
 * behind it, and returns WITHOUT synchronising: the copies of this step overlap
 * whatever is enqueued on `stream` next (another handle's step, or this handle's
 * next step once its outputs were read).  `slot` (0 .. PCL_HOST_SLOTS - 1) names
 * the completion event; pcl_host_wait(h, slot) blocks until the h_* buffers of
 * that call are valid.  Until then the caller must leave h_actions and the h_*
 * buffers alone, and must not call the synchronous step entry points on `h`.
 * With `crop` non-NULL the step is followed by pcl_crop(crop, d_crop, d_crop_state)
 * and h_view receives the crops u8 [B, crop rows, crop cols] instead of the
 * boards u8 [B, rows, pitch] — only the view the agent consumes crosses PCIe
 * (cropping.py:393-426 applied before the hand-off).  The crop spec is checked before
 * anything is enqueued: a spec pcl_crop refuses, and a tracking list that names a drape
 * (the curtains are not passed here: use pcl_crop_tracking), return their status
 * (PCL_ERR_UNSUPPORTED for the drape) with no env stepped. */
#define PCL_HOST_SLOTS 8
int pcl_step_host_async(pcl_handle* h, const int32_t* h_actions, int32_t* d_actions,
                        const pcl_outputs* out, const struct pcl_crop_spec* crop,
                        uint8_t* d_crop, int32_t* d_crop_state, uint8_t* h_view,
                        int32_t* h_reward, uint8_t* h_has_reward, float* h_discount,
                        uint8_t* h_done, int slot, void* stream);
int pcl_host_wait(pcl_handle* h, int slot);

/* Stand-alone renderer = Engine._render() + BaseObservationRenderer
 * (engine.py:737-759, rendering.py:98-179) over reference-layout inputs:
 * u8 backdrop [*, rows, pitch], byte curtains u8 [B, n_drapes, rows, pitch],
 * sprite records, per-env z-order u8 [B, n_sprites + n_drapes] of chars. */
int pcl_render(pcl_handle* h, const uint8_t* d_backdrop, int64_t backdrop_bstride,
               const uint8_t* d_curtains, const int32_t* d_sprites,
               const uint8_t* d_z_order, uint8_t* d_board, void* stream);

/* Byte-per-cell view of drape `drape_index`'s current curtain (Drape.curtain,
 * things.py:213-217): u8 [B, rows, pitch], the drape's plane of a one-character
 * pcl_layers call.  PCL_ERR_UNSUPPORTED where pcl_layers is; PCL_ERR_INVALID when
 * the bound state holds no curtain for that drape. */
int pcl_export_curtain(pcl_handle* h, int drape_index, uint8_t* d_out, void* stream);

/* Layers of BaseUnoccludedObservationRenderer (rendering.py:187-301, selected by
 * Engine(occlusion_in_layers=False), engine.py:564-570) for the whole batch: plane k
 * of d_out u8 [B, n_chars, rows, pitch] is 1 wherever the owner of chars[k] places it,
 * occluded or not — the backdrop where it holds that character, a drape's whole
 * curtain, a visible sprite's cell.  `chars` is a HOST array of n_chars <= 32 ASCII
 * codes.  PCL_ERR_UNSUPPORTED for programs whose drape curtain is implicit
 * (warehouse 'X', aperture, hello). */
int pcl_layers(pcl_handle* h, const uint8_t* chars, int32_t n_chars, uint8_t* d_out,
               void* stream);

/* ScrollingCropper.crop (cropping.py:393-426): track sprite `sprite_index`,
 * update the per-env window corner and copy the crop_rows x crop_cols window of
 * d_board into d_crop u8 [B, crop_rows, crop_cols].  The corner lives in
 * d_crop_state, i32 [B, 4] = (row, col, initialised, episode) owned by the
 * caller, one array per cropper object (zero-filled at creation); a window
 * re-initialises itself when the env's episode counter moves on, as
 * ScrollingCropper.set_engine does for a new Engine (cropping.py:375-391).
 * d_crop_state == NULL selects a single built-in cropper slot in the plot record.
 * sprite_index < 0 is a FixedCropper at (offset_rows, offset_cols).
 * Windows of more than PCL_MAX_CROP_CELLS cells are PCL_ERR_UNSUPPORTED at every cropper
 * entry point (the kernels divide a cell index by the width with a 16-bit-exact reciprocal). */
#define PCL_MAX_TRACK 4
#define PCL_MAX_CROP_CELLS 65535
typedef struct pcl_crop_spec {
  int32_t rows, cols;          /* window shape */
  int32_t sprite_index;        /* entity to track (a sprite) */
  int32_t pad_char;            /* ASCII code, or -1 for None */
  int32_t margin_rows, margin_cols; /* resolved scroll margins (cropping.py:362-373) */
  int32_t offset_rows, offset_cols; /* initial_offset */
  int32_t saccade;
  int32_t track[PCL_MAX_TRACK];     /* optional priority list (pcl_crop_tracking): k > 0 = sprite
                                       k - 1, k < 0 = drape -k - 1, 0 = end; all 0 = [sprite_index] */
} pcl_crop_spec;
int pcl_crop(pcl_handle* h, const pcl_crop_spec* crop, const uint8_t* d_board,
             uint8_t* d_crop, int32_t* d_crop_state, void* stream);

/* Attach ONE cropper to the handle: every later pcl_reset / pcl_step / pcl_run then also
 * writes the cropper's view of the new board into d_crop (u8 [B, rows, cols]) from INSIDE
 * the step kernel — what pcl_crop would produce if called right after the step, without
 * the second launch.  d_crop_state as for pcl_crop (NULL = the plot record's slot).
 * crop == NULL detaches.  Step programs without the epilogue (today every program but
 * PCL_PROG_SCROLLY_MAZE) and tracking lists that name drapes return PCL_ERR_UNSUPPORTED:
 * call pcl_crop after the step instead.  The buffers must outlive the attachment;
 * pcl_bind_state detaches.  pcl_step_host_async given the SAME spec, d_crop and
 * d_crop_state does not launch the cropper a second time. */
int pcl_attach_cropper(pcl_handle* h, const pcl_crop_spec* crop, uint8_t* d_crop,
                       int32_t* d_crop_state);

/* pcl_crop for a ScrollingCropper whose `to_track` names several entities
 * (cropping.py:544-598): the window follows the FIRST entry of crop->track that is
 * visible — a sprite that is visible, or a drape whose curtain has any cell, in
 * which case the position is (median row, median column) of its cells, truncated.
 * d_curtains[i] is the curtain of the drape named by track[i] as u8 [B, rows, pitch]
 * (what pcl_export_curtain writes); entries for sprites are ignored and may be
 * NULL.  Boards up to 128 x 128 when a drape is tracked. */
int pcl_crop_tracking(pcl_handle* h, const pcl_crop_spec* crop, const uint8_t* d_board,
                      uint8_t* d_crop, int32_t* d_crop_state,
                      const uint8_t* const* d_curtains, void* stream);

/* Observation post-processors as one table look-up per cell
 * (rendering.py:304-661): out[b, d, r, c] = table[board[b, r, c]][d].
 *   ObservationCharacterRepainter: depth 1, u8 table = the character mapping;
 *   ObservationToArray:            the value mapping (scalars or depth-vectors);
 *   ObservationToFeatureArray:     f32 one-hot, table[ch][d] = (ch == layers[d]).
 * d_table is [128, depth] of `dtype`, 1 <= depth <= 32 (callers split deeper
 * outputs into launches of <= 32 planes); d_valid u8 [128] marks characters the
 * mapping knows (NULL = all).  A cell holding a byte >= 128 gets zero elements.
 * An in-board cell whose byte is >= 128 or not valid sets *d_unknown (i32, may be
 * NULL) to 1 (upstream RuntimeError, rendering.py:520-526); pad columns are not
 * read.  Only the element size matters, the bits are copied: any 1-, 2-, 4- or
 * 8-byte type (bool, int8, float16, uint32, ...) fits the code of its size.
 * Output strides are in ELEMENTS, so any `permute` is just a stride choice. */
typedef struct pcl_observe_spec {
  int32_t depth;
  int32_t dtype;              /* 0 uint8, 1 int32, 2 float32, 3 int64, 4 float64,
                                 5 any 2-byte type (int16, uint16, float16) */
  int64_t stride_b, stride_d, stride_r, stride_c;
} pcl_observe_spec;
int pcl_observe(pcl_handle* h, const pcl_observe_spec* spec, const void* d_table,
                const uint8_t* d_valid, const uint8_t* d_board, void* d_out,
                int32_t* d_unknown, void* stream);

/* A cropper feeding a post-processor, in ONE launch from the board: pcl_crop_tracking
 * (crop, d_board, d_crop_state, d_curtains: same checks, same corner state, NULL = the plot
 * record's slot; the window moves exactly once per call whatever the depth) followed by
 * pcl_observe over the crop_rows x crop_cols window, without the crop ever being stored:
 *   out[b, d, jr, jc] = d_table[cell][d]
 * where cell is the window's byte (the pad character off the board).  The strides of
 * `spec` are in elements over (env, plane, window row, window column); any depth >= 1.
 * A window cell, pad included, holding a byte >= 128 or one d_valid does not mark sets
 * *d_unknown to 1 (upstream's RuntimeError for the cropped observation).
 * Un-occluded layers (games with occlusion_in_layers=False): with d_planes set, d_board
 * is not read; output plane d is source plane d_plane_of[d] (i32 [depth] on the device,
 * -1 = a plane of zeros) cut at the same window, and the cell is that plane's bit: 1 where
 * the plane's byte is non-zero, and off the board 1 exactly when d_plane_of[d] ==
 * pad_plane (the source plane of the pad character, or -1).  Source plane k of env b
 * starts at d_planes + b * plane_stride_b + k * plane_stride_d, rows plane_stride_r bytes
 * apart, one byte per column (pcl_layers' output, or any u8 / bool planes).  The table is
 * looked up at rows 0 and 1 then, and d_unknown is not set. */
int pcl_crop_observe(pcl_handle* h, const pcl_crop_spec* crop, const uint8_t* d_board,
                     int32_t* d_crop_state, const uint8_t* const* d_curtains,
                     const pcl_observe_spec* spec, const void* d_table, const uint8_t* d_valid,
                     const uint8_t* d_planes, const int32_t* d_plane_of, int32_t pad_plane,
                     int64_t plane_stride_b, int64_t plane_stride_d, int64_t plane_stride_r,
                     void* d_out, int32_t* d_unknown, void* stream);

/* Multi-GPU hand-off record (SURVEY.md 8e): everything one env contributes to the
 * per-step all-gather, packed so that ONE collective moves it all.
 *   d_packed u8 [B, record_bytes]; one record = view_bytes of the env's observation
 *   view (e.g. its 9x9 crop, row-major; d_view is u8 [B, view_bytes]), zero padding
 *   to a multiple of 4, then reward i32, discount f32, done u8, has_reward u8 and
 *   2 padding bytes; record_bytes = PCL_HANDOFF_RECORD_BYTES(view_bytes). */
#define PCL_HANDOFF_RECORD_BYTES(view_bytes) ((((view_bytes) + 3) & ~3) + 12)
int pcl_pack_handoff(pcl_handle* h, const uint8_t* d_view, int32_t view_bytes,
                     const pcl_outputs* out, uint8_t* d_packed, void* stream);

/* pcl_pack_handoff with the all-gather fused into the producing kernel: every
 * record is stored straight into the gather buffer of EVERY rank over NVLink
 * (peer-to-peer stores), so no collective library call sits between the step and
 * its consumers.  d_peer_bases (a HOST array of n_peers <= PCL_MAX_PEERS peer-mapped
 * device pointers, e.g. torch symmetric memory) are the bases of the ranks' gather
 * buffers u8 [rows, record_bytes]; this handle's env e lands in row first_row + e
 * of each.  The caller orders steps with a cross-GPU barrier (the records are
 * complete on every peer once this kernel has finished on every rank). */
#define PCL_MAX_PEERS 8
int pcl_pack_handoff_peers(pcl_handle* h, const uint8_t* d_view, int32_t view_bytes,
                           const pcl_outputs* out, uint8_t* const* d_peer_bases,
                           int32_t n_peers, int64_t first_row, void* stream);

/* ScrollingCropper.crop + pcl_pack_handoff_peers + the cross-GPU barrier in ONE
 * kernel (SURVEY.md 8e; cropping.py:393-426 for the view): every env's record —
 * its crop_rows x crop_cols window, zero padding to a multiple of 4, reward i32,
 * discount f32, done u8, has_reward u8, then zero padding up to `record_bytes` — is
 * stored with 16-byte stores into row first_row + env of EVERY rank's gather buffer
 * over NVLink (or once through `d_multicast`, the NVLS multicast mapping of those
 * buffers).  The last thread block to finish publishes this rank's step count in
 * every peer's flag array and waits until every peer has published the same count
 * here: when the kernel retires, half (step & 1) of the LOCAL gather buffer holds
 * all ranks' records of this step.  No collective call and no separate barrier
 * kernel; the step count lives in device memory (`d_local`), so the launch can be
 * captured in a CUDA graph.  Every rank must make the same sequence of calls.
 *   gather buffer of a rank: u8 [n_bufs, rows, record_bytes]  (parts alternate by step)
 *   flag array of a rank:    u32 [PCL_MAX_PEERS], zero-initialised; word s = steps
 *                            whose records from rank s have landed here
 *   d_local:                 u32 [2] zero-initialised device memory of this rank
 * record_bytes: multiple of 16, >= PCL_HANDOFF_RECORD_BYTES(crop rows * cols), <= 256. */
#define PCL_HANDOFF_LAG 1
#define PCL_HANDOFF_SIGNAL_KERNEL 2
typedef struct pcl_handoff {
  int32_t n_peers, rank;
  int32_t record_bytes;
  int64_t rows, first_row;
  uint8_t* d_peer_base[PCL_MAX_PEERS];   /* peer-mapped: every rank's gather buffer */
  uint32_t* d_peer_flags[PCL_MAX_PEERS]; /* peer-mapped: every rank's flag array   */
  uint8_t* d_multicast;                  /* multicast mapping of the gather buffers, or NULL */
  uint32_t* d_local;
  int32_t n_bufs;   /* parts of a gather buffer that alternate by step: 0 or 2 = two halves */
  int32_t mode;     /* bit flags:
                     * PCL_HANDOFF_LAG (1), split phase: signal this step but only wait for the
                     *   PREVIOUS one, so the cross-GPU wait leaves the critical path: when the call
                     *   for step s retires, part (s - 1) % n_bufs holds every rank's records of step
                     *   s - 1.  Needs n_bufs >= 3 (a peer one step ahead writes part (s + 1) % n_bufs
                     *   while part (s - 1) % n_bufs is being read); the last step is completed by any
                     *   host-level barrier after the stream has drained.
                     * PCL_HANDOFF_SIGNAL_KERNEL (2): the records kernel neither fences nor counts
                     *   blocks; a second, one-warp kernel behind it (the kernel boundary completes
                     *   the peer stores) publishes the flags and waits.  Measured faster than
                     *   1024 blocks each waiting for its NVLink acknowledgements. */
} pcl_handoff;
int pcl_crop_handoff(pcl_handle* h, const pcl_crop_spec* crop, const uint8_t* d_board,
                     int32_t* d_crop_state, const pcl_outputs* out, const pcl_handoff* x,
                     void* stream);

/* Copy the per-env latched error words (PCL_ENV_ERR_*) to d_out i32 [B]. */
int pcl_error_codes(pcl_handle* h, int32_t* d_out, void* stream);

/* Number of kernels this handle has launched so far. */
int pcl_launch_count(pcl_handle* h, int64_t* out);

const char* pcl_status_string(int status);
/* Text of the last CUDA failure behind a PCL_ERR_CUDA of this handle ("" if none);
 * valid until the next failing call on the handle. */
const char* pcl_last_error(pcl_handle* h);
int pcl_abi_version(void);
/* sizeof of the four structs that cross the boundary, for bindings to verify their
 * own layouts at load time: out[0..3] = pcl_spec, pcl_state, pcl_outputs, pcl_crop_spec. */
int pcl_struct_sizes(int32_t out[4]);

#ifdef __cplusplus
}
#endif
#endif  /* PCL_H_ */
