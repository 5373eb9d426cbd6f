// pcl_kernels.cuh — kernel parameter blocks, step-program descriptors, launch prototypes.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "../../include/pcl.h"

namespace pcl {

struct CropParams {
  int B, H, W, pitch, S;
  pcl_crop_spec crop;
  const int32_t* sprites;
  int32_t* plot;
  int32_t* state;                // i32 [B, 4] per-cropper corner state, or NULL
  const uint8_t* board;
  uint8_t* out;
  const uint8_t* curtains[PCL_MAX_TRACK];   // byte curtains of tracked drapes (or NULL)
  uint32_t cols_recip;           // floor(2^32 / crop.cols) + 1 (crop_params, api.cu)
};

// Everything a fused step kernel needs, by value (fits the 4 KB param space).
struct StepParams {
  int B, H, W, pitch;
  int PH, PW, PWW;               // Scrolly pattern rows/cols/words-per-row
  int BW;                        // words per bit-packed board-sized row
  int S, D;
  int auto_reset;
  int mode;                      // MODE_STEP / MODE_RESET
  int actions_per_env;
  int margin[PCL_MAX_DRAPES][2];
  uint8_t sprite_char[PCL_MAX_SPRITES];
  uint8_t drape_char[PCL_MAX_DRAPES];
  uint32_t impassable[PCL_MAX_SPRITES][4];
  int confined[PCL_MAX_SPRITES];
  int egocentric[PCL_MAX_SPRITES];
  int drape_kind[PCL_MAX_DRAPES];
  int program_arg[8];
  int n_scroll_groups;
  int sprite_group[PCL_MAX_SPRITES];
  int drape_group[PCL_MAX_DRAPES];
  int n_groups;
  int group_len[PCL_MAX_SPRITES + PCL_MAX_DRAPES];
  uint8_t group_chars[PCL_MAX_SPRITES + PCL_MAX_DRAPES];
  pcl_state st;
  pcl_outputs out;
  const int32_t* actions;        // i32 [B, actions_per_env] (MODE_STEP)
  const uint8_t* env_mask;       // u8 [B] or NULL (MODE_RESET)
  int has_cropper;               // pcl_attach_cropper: crop the new board as the kernel's epilogue
  CropParams cropper;            // (board is taken from `out` at launch time)
  const int32_t* code;           // device copy of the bytecode bound with pcl_bind_code, or NULL
  uint8_t* backdrop_live;        // pcl_bind_backdrop: u8 [B, H, pitch] live curtains, or NULL
  // Program::derive: device copies the program builds from the static level data bound
  // with pcl_bind_state, in formats only that program knows (indexed like the arrays they
  // come from: per level, or one copy when the stride is 0).
  const uint32_t* derived[3];
  int64_t derived_bstride[3];    // in words
  // Program::derive: per-env words the program keeps from one launch to the next (also in
  // the derived allocation, so every pcl_bind_state starts them afresh), or NULL.
  // scrolly_maze: what the board of each env was last drawn from.
  int32_t* render_key;
  // The handle's count of board-buffer changes: a launch whose out.d_board differs from
  // the previous launch's gets the next value, so each value names one buffer.
  uint32_t board_epoch;
};

// Launch with the programmatic-stream-serialisation attribute (the kernel calls
// griddepcontrol.wait before its first global access).
template <typename... Params, typename... Args>
cudaError_t launch_pdl(void (*kern)(Params...), int grid, int block, size_t smem, cudaStream_t s,
                       Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid); cfg.blockDim = dim3(block); cfg.dynamicSmemBytes = smem; cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, args...);
}

// A fused step kernel over p.B envs, one warp per env and `warps` envs per block,
// with `smem` bytes of dynamic shared memory per block; `pdl`: launch_pdl.
inline cudaError_t launch_step(void (*kern)(StepParams), const StepParams& p, int warps,
                               size_t smem, cudaStream_t s, bool pdl = false) {
  if (smem > 48 * 1024) {   // opt in per launch: the attribute is per device, handles are not
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  const int grid = (p.B + warps - 1) / warps;
  if (pdl) return launch_pdl(kern, grid, warps * 32, smem, s, p);
  kern<<<grid, warps * 32, smem, s>>>(p);
  return cudaGetLastError();
}

// Where a drape's curtain lives in the bound state (resolve_curtain, api.cu): nowhere the
// layers kernel can read (held implicitly by the program), bit rows of the board
// (d_bits), or a window of its Scrolly pattern (d_pattern) at the drape's corner, whose
// drape record may name one stale cell (kStaleWindow: AUX0 / AUX1).
enum class CurtainAt { kNone, kBits, kPatternWindow, kStaleWindow };

// Everything the C boundary needs to know about one step program.  Each program's .cu
// file defines its descriptor beside its kernel; api.cu maps PCL_PROG_* ids to them.
struct Program {
  int (*check_spec)(const pcl_spec&);                      // PCL_OK / _INVALID / _UNSUPPORTED
  int (*check_state)(const pcl_spec&, const pcl_state&);   // nullptr: only the common records
  CurtainAt (*curtain)(const pcl_spec&, int drape);        // nullptr: every drape kNone
  cudaError_t (*launch)(const StepParams&, cudaStream_t);  // nullptr: nothing to step
  int (*actions_per_env)(const pcl_spec&);                 // nullptr: 1
  bool float_reward;             // rewards go to pcl_outputs.d_reward_f64, not d_reward
  bool crop_epilogue;            // the step kernel runs an attached cropper (pcl_attach_cropper)
  bool scroll_groups;            // accepts more than one scrolling group
  // Programs that run bytecode (pcl_bind_code): checks the host words against the spec,
  // PCL_OK / PCL_ERR_INVALID.  nullptr: the program takes no code.
  int (*check_code)(const pcl_spec&, const int32_t* words, int n_words);
  bool float_reward_arg0;        // rewards are float64 when spec.program_arg[0] != 0
  // Called before the first step or reset after each pcl_bind_state: builds
  // StepParams::derived* from the bound state for a handle of `batch` envs, in one device
  // allocation returned in *owned (the handle frees it when it rebuilds and at
  // pcl_destroy).  May synchronise the device.  nullptr: the program derives nothing.
  int (*derive)(const pcl_spec&, const pcl_state&, int batch, StepParams* base, void** owned);
};
extern const Program kScrollyMaze, kWarehouse, kMarauders, kFixture, kBetterScrolly, kClassics,
    kAperture, kOrdeal, kHello, kApprehend, kShockwave, kTMaze, kCompiled, kBoxWorld,
    kCuedCatch, kSequenceRecall;

// Host-side helpers of the programs' check_spec.
inline bool chars_are(const uint8_t* got, int n, const char* want) {
  if ((int)strlen(want) != n) return false;
  for (int i = 0; i < n; ++i) if (got[i] != (uint8_t)want[i]) return false;
  return true;
}

// The set `want` as a 128-bit ASCII mask equals `got`?
inline bool set_is(const uint32_t (&got)[4], const char* want) {
  uint32_t m[4] = {0, 0, 0, 0};
  for (const char* c = want; *c; ++c) m[(*c >> 5) & 3] |= 1u << (*c & 31);
  return m[0] == got[0] && m[1] == got[1] && m[2] == got[2] && m[3] == got[3];
}

inline int groups_are(const pcl_spec& s, const char* flat, const int* lens, int n) {
  if (s.n_groups != n) return 0;
  int k = 0;
  for (int g = 0; g < n; ++g) {
    if (s.group_len[g] != lens[g]) return 0;
    for (int i = 0; i < lens[g]; ++i, ++k)
      if (s.group_chars[k] != (uint8_t)flat[k]) return 0;
  }
  return 1;
}

// bits_words holds a bit-packed board row (d_bits) and one word more.
inline bool bit_rows_fit(const pcl_spec& s) { return s.bits_words >= (s.cols + 31) / 32 + 1; }

// Scrolly d's margins (-1 = None) overlap no more than half of the board (drapes.py:350-364).
inline bool margins_fit(const pcl_spec& s, int d) {
  const int mr = s.margins[d][0], mc = s.margins[d][1];
  return !(mr >= 0 && (mc - 1 >= s.cols - mc || mr - 1 >= s.rows - mr));
}

// Program::curtain of programs that keep every drape in d_bits.
inline CurtainAt curtain_bits(const pcl_spec&, int) { return CurtainAt::kBits; }

struct RenderParams {
  int B, H, W, pitch, S, D;
  const uint8_t* backdrop; int64_t backdrop_bstride;
  const uint8_t* curtains;       // u8 [B, D, H, pitch]
  const int32_t* sprites;        // i32 [B, S, 8]
  const uint8_t* z_order;        // u8 [B, S + D] chars
  uint8_t sprite_char[PCL_MAX_SPRITES];
  uint8_t drape_char[PCL_MAX_DRAPES];
  uint8_t* board;                // u8 [B, H, pitch]
};
cudaError_t launch_render(const RenderParams& p, cudaStream_t s);

// Unoccluded layers (rendering.py:187-301): one mask per requested character.
#define PCL_MAX_LAYER_CHARS 32
struct LayersParams {
  int B, H, W, pitch, S, D, n_chars;
  uint8_t chars[PCL_MAX_LAYER_CHARS];
  int8_t sprite_of[PCL_MAX_LAYER_CHARS];   // sprite index painting that char, or -1
  int8_t drape_of[PCL_MAX_LAYER_CHARS];    // drape index painting that char, or -1
  // per drape: where its curtain lives in the packed state, as the program's
  // Program::curtain says (resolve_curtain, api.cu)
  const uint32_t* bits[PCL_MAX_DRAPES]; int64_t bits_bstride[PCL_MAX_DRAPES];
  int row_words[PCL_MAX_DRAPES];           // uint32 words per bit row
  int scrolly[PCL_MAX_DRAPES];             // 1: window of a pattern at the drape's corner
  int per_level[PCL_MAX_DRAPES];           // 1: `bits` is static per-level data
  int stale_slot[PCL_MAX_DRAPES];          // 1: the drape record's AUX0/1 hold a stale cell
  const uint8_t* backdrop; int64_t backdrop_bstride;
  const int32_t* level;
  const int32_t* sprites;
  const int32_t* drapes;
  uint8_t* out;                            // u8 [B, n_chars, H, pitch]
  int backdrop_per_env;                    // 1: `backdrop` is indexed by env, not level (live)
};
cudaError_t launch_layers(const LayersParams& p, cudaStream_t s);

struct ObserveParams {
  int B, H, W, pitch, depth, dtype;
  int words;                     // words per element: 2 for 8- and 2-byte elements
  int64_t stride_b, stride_d, stride_r, stride_c;   // in words (u32, or bytes for dtype 0 / 5)
  const void* table;             // [128, depth]
  const uint8_t* valid;          // u8 [128] or NULL
  const uint8_t* board;          // u8 [B, H, pitch]
  void* out;
  int32_t* unknown;              // i32 [1] or NULL
};
cudaError_t launch_observe(const ObserveParams& p, cudaStream_t s);

cudaError_t launch_crop(const CropParams& p, cudaStream_t s);

// Exchange state of the fused crop + hand-off kernel (pcl_crop_handoff).
struct HandoffParams {
  int n_peers, rank, record_bytes;
  int64_t rows;                  // records per half of a gather buffer
  int64_t first_row;             // this rank's first row
  uint8_t* peer_base[PCL_MAX_PEERS];    // peer-mapped bases of every rank's gather buffer (2 halves)
  uint32_t* peer_flags[PCL_MAX_PEERS];  // peer-mapped flag arrays u32 [PCL_MAX_PEERS] of every rank
  uint8_t* multicast;            // NVLS multicast mapping of the gather buffers, or NULL
  uint32_t* local;               // device-local u32 [2]: steps done, block ticket
  int n_bufs, lag;               // parts of the gather buffer; 1 = wait for the previous step only
  int signal_kernel;             // 1: a second one-warp kernel publishes and waits (no fences here)
  pcl_outputs out;
};
cudaError_t launch_crop_handoff(const CropParams& p, const HandoffParams& x, cudaStream_t s);

struct PackParams {
  int B, view_bytes, record_bytes;
  const uint8_t* view;           // u8 [B, view_bytes]
  pcl_outputs out;
  uint8_t* packed;               // u8 [B, record_bytes] (n_peers == 0)
  int n_peers;                   // > 0: store into every peer's gather buffer instead
  int64_t first_row;
  uint8_t* peers[PCL_MAX_PEERS];
};
cudaError_t launch_pack_handoff(const PackParams& p, cudaStream_t s);

}  // namespace pcl
