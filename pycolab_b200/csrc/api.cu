// api.cu — the extern "C" boundary declared in include/pcl.h.
#include <cuda_runtime.h>
#include <stdio.h>
#include <string.h>

#include <new>

#include <nvtx3/nvToolsExt.h>   // header-only NVTX v3: ranges show up in nsys / ncu timelines

#include "pcl_device.cuh"
#include "pcl_kernels.cuh"


struct pcl_handle {
  pcl_spec spec;
  const pcl::Program* program;   // the descriptor of spec.program
  int batch;
  int device;
  int bound;
  int actions_per_env;
  pcl_state st;
  long long launches;
  pcl::StepParams base;          // everything fill_params derives from spec + state, built once at bind
  char last_error[256];          // text of the last failed CUDA call (pcl_last_error)
  // pcl_step_host_async: a copy stream so that the D2H of one step overlaps the next kernel
  cudaStream_t copy_stream;
  cudaEvent_t ev_step[PCL_HOST_SLOTS];   // step kernel finished (compute stream)
  cudaEvent_t ev_done[PCL_HOST_SLOTS];   // host buffers of that slot are valid (copy stream)
  int host_ready;
  int pending_slot;              // slot of this handle's last async step whose D2H may still run, or -1
  // pcl_bind_code: the checked host words, and their device copy made at the next launch
  int32_t* code_host;
  int code_words;
  int32_t* code_dev;
  int code_dev_words;            // words the device buffer holds room for
  int code_stale;                // code_host changed since the upload
  uint8_t* backdrop_live;        // pcl_bind_backdrop, or NULL
  // Program::derive: its allocation for the bound state, and whether the state was bound
  // since it was built
  void* derived_dev;
  int derive_stale;
  // StepParams::board_epoch: the board buffer of the last launch, and its epoch
  const uint8_t* last_board;
  uint32_t board_epoch;
};

namespace {

using pcl::StepParams;

// One NVTX range per boundary call (a no-op costing a pointer test when no tool
// is attached); the ranges name the reference call each entry point stands for.
struct Range {
  explicit Range(const char* name) { nvtxRangePushA(name); }
  ~Range() { nvtxRangePop(); }
};

// Remember what failed: PCL_ERR_CUDA alone says nothing (pcl_last_error).
int cuda_failed(pcl_handle* h, cudaError_t e, const char* what) {
  if (h) snprintf(h->last_error, sizeof(h->last_error), "%s: %s (%s)", what,
                  cudaGetErrorString(e), cudaGetErrorName(e));
  return PCL_ERR_CUDA;
}

#define PCL_CUDA(h, call)                                        \
  do {                                                           \
    cudaError_t e_ = (call);                                     \
    if (e_ != cudaSuccess) return cuda_failed((h), e_, #call);   \
  } while (0)

int accept_any(const pcl_spec&) { return PCL_OK; }

// No step program: a handle for pcl_render / pcl_crop only; its steps are refused.
const pcl::Program kNone = {accept_any, nullptr, nullptr, nullptr, nullptr,
                            /*float_reward=*/false, /*crop_epilogue=*/false,
                            /*scroll_groups=*/false};

const struct {
  int id;
  const pcl::Program* program;
} kPrograms[] = {
    {PCL_PROG_NONE, &kNone},
    {PCL_PROG_SCROLLY_MAZE, &pcl::kScrollyMaze},
    {PCL_PROG_WAREHOUSE, &pcl::kWarehouse},
    {PCL_PROG_MARAUDERS, &pcl::kMarauders},
    {PCL_PROG_FIXTURE, &pcl::kFixture},
    {PCL_PROG_BETTER_SCROLLY, &pcl::kBetterScrolly},
    {PCL_PROG_CLASSICS, &pcl::kClassics},
    {PCL_PROG_APERTURE, &pcl::kAperture},
    {PCL_PROG_ORDEAL, &pcl::kOrdeal},
    {PCL_PROG_HELLO, &pcl::kHello},
    {PCL_PROG_APPREHEND, &pcl::kApprehend},
    {PCL_PROG_SHOCKWAVE, &pcl::kShockwave},
    {PCL_PROG_T_MAZE, &pcl::kTMaze},
    {PCL_PROG_COMPILED, &pcl::kCompiled},
    {PCL_PROG_BOX_WORLD, &pcl::kBoxWorld},
    {PCL_PROG_CUED_CATCH, &pcl::kCuedCatch},
    {PCL_PROG_SEQUENCE_RECALL, &pcl::kSequenceRecall},
};

// The descriptor of program `id`, or nullptr for an id this build does not know.
const pcl::Program* program_of(int id) {
  for (const auto& row : kPrograms) if (row.id == id) return row.program;
  return nullptr;
}

// Each program is lowered for one entity layout; anything else is a valid
// pycolab game that this build does not accelerate.
int validate(const pcl_spec& s) {
  const pcl::Program* prog = program_of(s.program);
  if (s.abi_version != PCL_ABI_VERSION) return PCL_ERR_INVALID;
  if (s.rows <= 0 || s.cols <= 0 || s.pitch < s.cols || (s.pitch & 15)) return PCL_ERR_INVALID;
  if (s.n_sprites < 0 || s.n_sprites > PCL_MAX_SPRITES) return PCL_ERR_INVALID;
  if (s.n_drapes < 0 || s.n_drapes > PCL_MAX_DRAPES) return PCL_ERR_INVALID;
  {
    // Scrolling groups: every entity names one of the declared groups; only
    // programs that keep more than one group's blackboard accept several.
    const int ng = s.n_scroll_groups < 1 ? 1 : s.n_scroll_groups;
    if (ng > PCL_MAX_SCROLL_GROUPS) return PCL_ERR_UNSUPPORTED;
    if (ng > 1 && !(prog && prog->scroll_groups)) return PCL_ERR_UNSUPPORTED;
    for (int i = 0; i < s.n_sprites; ++i)
      if (s.sprite_group[i] < 0 || s.sprite_group[i] >= ng) return PCL_ERR_INVALID;
    for (int i = 0; i < s.n_drapes; ++i)
      if (s.drape_group[i] < 0 || s.drape_group[i] >= ng) return PCL_ERR_INVALID;
  }
  return prog ? prog->check_spec(s) : PCL_ERR_UNSUPPORTED;
}

void fill_params(const pcl_handle* h, StepParams* p) {
  const pcl_spec& s = h->spec;
  memset(p, 0, sizeof(*p));
  p->B = h->batch; p->H = s.rows; p->W = s.cols; p->pitch = s.pitch;
  p->PH = s.pattern_rows; p->PW = s.pattern_cols; p->PWW = s.pattern_words;
  p->BW = s.bits_words;
  p->S = s.n_sprites; p->D = s.n_drapes;
  p->auto_reset = s.auto_reset;
  p->actions_per_env = h->actions_per_env;
  memcpy(p->margin, s.margins, sizeof(p->margin));
  memcpy(p->sprite_char, s.sprite_char, sizeof(p->sprite_char));
  memcpy(p->drape_char, s.drape_char, sizeof(p->drape_char));
  memcpy(p->impassable, s.impassable, sizeof(p->impassable));
  memcpy(p->confined, s.sprite_confined, sizeof(p->confined));
  memcpy(p->egocentric, s.sprite_egocentric, sizeof(p->egocentric));
  memcpy(p->drape_kind, s.drape_kind, sizeof(p->drape_kind));
  memcpy(p->program_arg, s.program_arg, sizeof(p->program_arg));
  p->n_scroll_groups = s.n_scroll_groups < 1 ? 1 : s.n_scroll_groups;
  memcpy(p->sprite_group, s.sprite_group, sizeof(p->sprite_group));
  memcpy(p->drape_group, s.drape_group, sizeof(p->drape_group));
  p->n_groups = s.n_groups;
  memcpy(p->group_len, s.group_len, sizeof(p->group_len));
  memcpy(p->group_chars, s.group_chars, sizeof(p->group_chars));
  p->st = h->st;
  p->code = h->code_dev;
  p->backdrop_live = h->backdrop_live;
}

// Does the handle's Backdrop run compiled code on a live curtain (pcl_bind_backdrop)?
bool live_backdrop(const pcl_spec& s) {
  return s.program == PCL_PROG_COMPILED && s.program_arg[4] != 0;
}

int launch(pcl_handle* h, StepParams p, cudaStream_t stream) {
  if (!h->program->launch) return PCL_ERR_UNSUPPORTED;
  if (p.out.d_board != h->last_board) {
    h->last_board = p.out.d_board;
    h->board_epoch += 1;
  }
  p.board_epoch = h->board_epoch;
  const cudaError_t e = h->program->launch(p, stream);
  if (e != cudaSuccess) return cuda_failed(h, e, "step kernel launch");
  h->launches += 1;              // only launches that were accepted count
  return PCL_OK;
}

// Status of a non-step kernel launch; counts it when it went through.
int launched(pcl_handle* h, cudaError_t e, const char* what) {
  if (e != cudaSuccess) return cuda_failed(h, e, what);
  h->launches += 1;
  return PCL_OK;
}

// The per-env outputs every step writes and every hand-off record carries.
bool outputs_set(const pcl_outputs& out) {
  return out.d_reward && out.d_has_reward && out.d_discount && out.d_done;
}

// Are this handle's rewards float64 (pcl_outputs.d_reward_f64)?
bool float_rewards(const pcl_handle* h) {
  return h->program->float_reward || (h->program->float_reward_arg0 && h->spec.program_arg[0]);
}

// Copy the bound bytecode to the device if it changed since the last launch, in order on
// `s` (the stream of the launch about to use it), and wait for the copy: once this
// returns, a launch on any stream reads complete code.  Rebinding first waits for the
// device, so no kernel still running the old code sees its buffer change.  The copy
// carries two zero words more, so the kernel may read an operand word past a final RET.
int upload_code(pcl_handle* h, cudaStream_t s) {
  if (!h->code_stale) return PCL_OK;
  if (h->code_dev) PCL_CUDA(h, cudaDeviceSynchronize());
  if (h->code_dev_words < h->code_words + 2) {
    if (h->code_dev) PCL_CUDA(h, cudaFree(h->code_dev));
    h->code_dev = nullptr;
    h->code_dev_words = 0;
    h->base.code = nullptr;
    PCL_CUDA(h, cudaMalloc(&h->code_dev, (h->code_words + 2) * sizeof(int32_t)));
    h->code_dev_words = h->code_words + 2;
  }
  PCL_CUDA(h, cudaMemsetAsync(h->code_dev, 0, h->code_dev_words * sizeof(int32_t), s));
  PCL_CUDA(h, cudaMemcpyAsync(h->code_dev, h->code_host, h->code_words * sizeof(int32_t),
                              cudaMemcpyHostToDevice, s));
  PCL_CUDA(h, cudaStreamSynchronize(s));
  h->base.code = h->code_dev;
  h->code_stale = 0;
  return PCL_OK;
}

// Build the program's derived copies of the state bound since the last launch (the
// first launch after pcl_bind_state reads the static level data; binding itself touches
// no device memory).  Launches still in flight may read the previous copies: wait first.
int derive_state(pcl_handle* h) {
  if (!h->derive_stale) return PCL_OK;
  if (h->derived_dev) {
    PCL_CUDA(h, cudaDeviceSynchronize());
    PCL_CUDA(h, cudaFree(h->derived_dev));
    h->derived_dev = nullptr;
  }
  const int r = h->program->derive(h->spec, h->st, h->batch, &h->base, &h->derived_dev);
  if (r == PCL_ERR_CUDA) return cuda_failed(h, cudaGetLastError(), "Program::derive");
  if (r != PCL_OK) return r;
  h->derive_stale = 0;
  return PCL_OK;
}

// Everything a step or reset on `s` needs is in place; uploads bound code and builds
// derived copies on the way.
int check_ready(pcl_handle* h, const pcl_outputs* out, cudaStream_t s) {
  if (!h || !out) return PCL_ERR_INVALID;
  if (!h->bound) return PCL_ERR_UNBOUND;
  if (h->program->check_code && !h->code_host) return PCL_ERR_UNBOUND;
  if (live_backdrop(h->spec) && !h->backdrop_live) return PCL_ERR_UNBOUND;
  if (!out->d_board || !outputs_set(*out)) return PCL_ERR_INVALID;
  if (float_rewards(h) && !out->d_reward_f64) return PCL_ERR_INVALID;
  const int r = derive_state(h);
  if (r != PCL_OK) return r;
  return h->program->check_code ? upload_code(h, s) : PCL_OK;
}

__global__ void gather_errors(const int32_t* plot, int32_t* out, int B) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < B) out[i] = plot[(int64_t)i * PCL_PLOT_WORDS + PCL_P_ERROR];
}

}  // namespace

extern "C" {

int pcl_abi_version(void) { return PCL_ABI_VERSION; }

int pcl_struct_sizes(int32_t out[4]) {
  if (!out) return PCL_ERR_INVALID;
  out[0] = (int32_t)sizeof(pcl_spec); out[1] = (int32_t)sizeof(pcl_state);
  out[2] = (int32_t)sizeof(pcl_outputs); out[3] = (int32_t)sizeof(pcl_crop_spec);
  return PCL_OK;
}

const char* pcl_status_string(int status) {
  switch (status) {
    case PCL_OK: return "ok";
    case PCL_ERR_INVALID: return "invalid argument or malformed spec";
    case PCL_ERR_UNSUPPORTED: return "game not lowered to a device program";
    case PCL_ERR_CUDA: return "CUDA runtime error";
    case PCL_ERR_UNBOUND: return "pcl_bind_state (or, for PCL_PROG_COMPILED, pcl_bind_code) has not been called";
    case PCL_ERR_NOMEM: return "out of memory";
    default: return "unknown status";
  }
}

int pcl_create(const pcl_spec* spec, int batch, int device, pcl_handle** out) {
  if (!spec || !out || batch <= 0) return PCL_ERR_INVALID;
  const int v = validate(*spec);
  if (v != PCL_OK) return v;
  if (device >= 0 && cudaSetDevice(device) != cudaSuccess) return PCL_ERR_CUDA;
  pcl_handle* h = new (std::nothrow) pcl_handle();
  if (!h) return PCL_ERR_NOMEM;
  h->spec = *spec;
  h->program = program_of(spec->program);
  h->batch = batch;
  h->device = device;
  h->bound = 0;
  h->actions_per_env = h->program->actions_per_env ? h->program->actions_per_env(*spec) : 1;
  h->launches = 0;
  h->last_error[0] = 0;
  h->host_ready = 0;
  h->pending_slot = -1;
  h->code_host = nullptr;
  h->code_words = 0;
  h->code_dev = nullptr;
  h->code_dev_words = 0;
  h->code_stale = 0;
  h->backdrop_live = nullptr;
  h->derived_dev = nullptr;
  h->derive_stale = 0;
  h->last_board = nullptr;
  h->board_epoch = 0;
  *out = h;
  return PCL_OK;
}

int pcl_destroy(pcl_handle* h) {
  if (h && h->host_ready) {
    for (int i = 0; i < PCL_HOST_SLOTS; ++i) {
      cudaEventDestroy(h->ev_step[i]);
      cudaEventDestroy(h->ev_done[i]);
    }
    cudaStreamDestroy(h->copy_stream);
  }
  if (h) {
    if (h->code_dev) cudaFree(h->code_dev);
    if (h->derived_dev) cudaFree(h->derived_dev);
    delete[] h->code_host;
  }
  delete h;
  return PCL_OK;
}

const char* pcl_last_error(pcl_handle* h) { return h ? h->last_error : ""; }

int pcl_bind_state(pcl_handle* h, const pcl_state* st) {
  if (!h || !st) return PCL_ERR_INVALID;
  if (!st->d_backdrop || !st->d_plot || !st->d_plot_init) return PCL_ERR_INVALID;
  // A game may have no sprites at all (engine_test.py:578-640 renders one drape).
  if (h->spec.n_sprites > 0 && (!st->d_sprites || !st->d_sprites_init)) return PCL_ERR_INVALID;
  if (h->spec.n_drapes > 0 && (!st->d_drapes || !st->d_drapes_init)) return PCL_ERR_INVALID;
  if (h->spec.n_scroll_groups > 1 && (!st->d_groups || !st->d_groups_init)) return PCL_ERR_INVALID;
  if (h->program->check_state) {
    const int r = h->program->check_state(h->spec, *st);
    if (r != PCL_OK) return r;
  }
  h->st = *st;
  fill_params(h, &h->base);      // the per-step calls only patch mode / actions / outputs
  h->derive_stale = h->program->derive != nullptr;
  h->bound = 1;
  return PCL_OK;
}

int pcl_bind_code(pcl_handle* h, const int32_t* h_code, int32_t n_words) {
  if (!h || !h_code) return PCL_ERR_INVALID;
  if (!h->program->check_code) return PCL_ERR_UNSUPPORTED;
  if (n_words < 1 || n_words > PCL_MAX_CODE_WORDS) return PCL_ERR_INVALID;
  const int r = h->program->check_code(h->spec, h_code, n_words);
  if (r != PCL_OK) return r;
  int32_t* copy = new (std::nothrow) int32_t[n_words];
  if (!copy) return PCL_ERR_NOMEM;
  memcpy(copy, h_code, n_words * sizeof(int32_t));
  delete[] h->code_host;
  h->code_host = copy;
  h->code_words = n_words;
  h->code_stale = 1;
  return PCL_OK;
}

int pcl_bind_backdrop(pcl_handle* h, uint8_t* d_backdrop_live) {
  if (!h || !d_backdrop_live || !live_backdrop(h->spec)) return PCL_ERR_INVALID;
  h->backdrop_live = d_backdrop_live;
  h->base.backdrop_live = d_backdrop_live;   // pcl_bind_state's fill_params copies it too
  return PCL_OK;
}

int pcl_reset(pcl_handle* h, const uint8_t* d_env_mask, const pcl_outputs* out, void* stream) {
  Range nvtx_range("pcl_reset (Engine.its_showtime)");
  const int r = check_ready(h, out, (cudaStream_t)stream);
  if (r != PCL_OK) return r;
  StepParams p = h->base;
  p.mode = pcl::MODE_RESET;
  p.env_mask = d_env_mask;
  p.out = *out;
  return launch(h, p, (cudaStream_t)stream);
}

int pcl_step(pcl_handle* h, const int32_t* d_actions, const pcl_outputs* out, void* stream) {
  Range nvtx_range("pcl_step (Engine.play)");
  const int r = check_ready(h, out, (cudaStream_t)stream);
  if (r != PCL_OK) return r;
  if (!d_actions) return PCL_ERR_INVALID;
  StepParams p = h->base;
  p.mode = pcl::MODE_STEP;
  p.actions = d_actions;
  p.out = *out;
  return launch(h, p, (cudaStream_t)stream);
}

int pcl_run(pcl_handle* h, const int32_t* d_actions, int steps, const pcl_outputs* out,
            void* stream) {
  Range nvtx_range("pcl_run");
  const int r = check_ready(h, out, (cudaStream_t)stream);
  if (r != PCL_OK) return r;
  if (!d_actions || steps < 0) return PCL_ERR_INVALID;
  StepParams p = h->base;
  p.mode = pcl::MODE_STEP;
  p.out = *out;
  for (int t = 0; t < steps; ++t) {
    p.actions = d_actions + (int64_t)t * h->batch * h->actions_per_env;
    const int e = launch(h, p, (cudaStream_t)stream);
    if (e != PCL_OK) return e;
  }
  return PCL_OK;
}

int pcl_run_many(pcl_handle* const* handles, int n_handles, const int32_t* const* d_actions,
                 const pcl_outputs* const* outs, int steps, void* stream) {
  Range nvtx_range("pcl_run_many");
  if (!handles || !d_actions || !outs || n_handles < 1 || steps < 0) return PCL_ERR_INVALID;
  for (int i = 0; i < n_handles; ++i) {
    const int r = check_ready(handles[i], outs[i], (cudaStream_t)stream);
    if (r != PCL_OK) return r;
  }
  for (int t = 0; t < steps; ++t) {
    if (!d_actions[t]) return PCL_ERR_INVALID;
    pcl_handle* h = handles[t % n_handles];
    StepParams p = h->base;
    p.mode = pcl::MODE_STEP;
    p.out = *outs[t % n_handles];
    p.actions = d_actions[t];
    const int e = launch(h, p, (cudaStream_t)stream);
    if (e != PCL_OK) return e;
  }
  return PCL_OK;
}

namespace {

// H2D of the action words, then the step, both on `s`.
int step_host_enqueue(pcl_handle* h, const int32_t* h_actions, int32_t* d_actions,
                      const pcl_outputs* out, cudaStream_t s) {
  const size_t B = (size_t)h->batch;
  PCL_CUDA(h, cudaMemcpyAsync(d_actions, h_actions, B * h->actions_per_env * sizeof(int32_t),
                              cudaMemcpyHostToDevice, s));
  return pcl_step(h, d_actions, out, (void*)s);
}

int copy_outputs(pcl_handle* h, const pcl_outputs* out, const uint8_t* d_view, size_t view_bytes,
                 uint8_t* h_view, int32_t* h_reward, uint8_t* h_has_reward, float* h_discount,
                 uint8_t* h_done, cudaStream_t s) {
  const size_t B = (size_t)h->batch;
  if (h_view) PCL_CUDA(h, cudaMemcpyAsync(h_view, d_view, view_bytes, cudaMemcpyDeviceToHost, s));
  if (h_reward) PCL_CUDA(h, cudaMemcpyAsync(h_reward, out->d_reward, B * 4, cudaMemcpyDeviceToHost, s));
  if (h_has_reward)
    PCL_CUDA(h, cudaMemcpyAsync(h_has_reward, out->d_has_reward, B, cudaMemcpyDeviceToHost, s));
  if (h_discount)
    PCL_CUDA(h, cudaMemcpyAsync(h_discount, out->d_discount, B * 4, cudaMemcpyDeviceToHost, s));
  if (h_done) PCL_CUDA(h, cudaMemcpyAsync(h_done, out->d_done, B, cudaMemcpyDeviceToHost, s));
  return PCL_OK;
}

int host_pipeline_ready(pcl_handle* h) {
  if (h->host_ready) return PCL_OK;
  PCL_CUDA(h, cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking));
  for (int i = 0; i < PCL_HOST_SLOTS; ++i) {
    PCL_CUDA(h, cudaEventCreateWithFlags(&h->ev_step[i], cudaEventDisableTiming));
    PCL_CUDA(h, cudaEventCreateWithFlags(&h->ev_done[i], cudaEventDisableTiming));
  }
  h->host_ready = 1;
  return PCL_OK;
}

// cropping.py:362-391: what a ScrollingCropper / FixedCropper accepts, for every
// cropper entry point.
int crop_spec_ok(const pcl_handle* h, const pcl_crop_spec* crop) {
  if (crop->rows <= 0 || crop->cols <= 0) return PCL_ERR_INVALID;
  // sprite_index names the tracked sprite only when no priority list is given (a
  // cropper may track a drape in a game without sprites).
  if (crop->track[0] == 0 && crop->sprite_index >= h->spec.n_sprites) return PCL_ERR_INVALID;
  if (crop->sprite_index >= 0 &&
      (2 * crop->margin_rows >= crop->rows || 2 * crop->margin_cols >= crop->cols))
    return PCL_ERR_INVALID;                                  // cropping.py:374-380
  if (crop->pad_char < 0 && (crop->rows > h->spec.rows || crop->cols > h->spec.cols))
    return PCL_ERR_INVALID;                                  // cropping.py:384-391
  for (int i = 0; i < PCL_MAX_TRACK && crop->track[i] != 0; ++i) {
    if (crop->sprite_index < 0) return PCL_ERR_INVALID;      // a FixedCropper tracks nothing
    if (crop->track[i] > h->spec.n_sprites || crop->track[i] < -h->spec.n_drapes)
      return PCL_ERR_INVALID;                                // no such sprite / drape
  }
  // A legal window upstream, but crop_word's reciprocal division is exact only below it.
  if ((int64_t)crop->rows * crop->cols > PCL_MAX_CROP_CELLS) return PCL_ERR_UNSUPPORTED;
  return PCL_OK;
}

bool tracks_drape(const pcl_crop_spec* crop) {
  for (int i = 0; i < PCL_MAX_TRACK && crop->track[i] != 0; ++i)
    if (crop->track[i] < 0) return true;
  return false;
}

}  // namespace

int pcl_step_host(pcl_handle* h, const int32_t* h_actions, int32_t* d_actions,
                  const pcl_outputs* out, uint8_t* h_board, int32_t* h_reward,
                  uint8_t* h_has_reward, float* h_discount, uint8_t* h_done, void* stream) {
  Range nvtx_range("pcl_step_host");
  const int r = check_ready(h, out, (cudaStream_t)stream);
  if (r != PCL_OK) return r;
  if (float_rewards(h)) return PCL_ERR_UNSUPPORTED;     // h_reward is int32
  if (!h_actions || !d_actions) return PCL_ERR_INVALID;
  cudaStream_t s = (cudaStream_t)stream;
  const size_t plane = (size_t)h->spec.rows * h->spec.pitch;
  int e = step_host_enqueue(h, h_actions, d_actions, out, s);
  if (e != PCL_OK) return e;
  e = copy_outputs(h, out, out->d_board, (size_t)h->batch * plane, h_board, h_reward, h_has_reward,
                   h_discount, h_done, s);
  if (e != PCL_OK) return e;
  PCL_CUDA(h, cudaStreamSynchronize(s));
  return PCL_OK;
}

int pcl_step_host_async(pcl_handle* h, const int32_t* h_actions, int32_t* d_actions,
                        const pcl_outputs* out, const pcl_crop_spec* crop, uint8_t* d_crop,
                        int32_t* d_crop_state, uint8_t* h_view, int32_t* h_reward,
                        uint8_t* h_has_reward, float* h_discount, uint8_t* h_done, int slot,
                        void* stream) {
  Range nvtx_range("pcl_step_host_async");
  const int r = check_ready(h, out, (cudaStream_t)stream);
  if (r != PCL_OK) return r;
  if (float_rewards(h)) return PCL_ERR_UNSUPPORTED;     // h_reward is int32
  if (!h_actions || !d_actions || slot < 0 || slot >= PCL_HOST_SLOTS) return PCL_ERR_INVALID;
  if (crop && !d_crop) return PCL_ERR_INVALID;
  if (crop) {                    // refuse the crop before the step, not after it
    const int ok = crop_spec_ok(h, crop);
    if (ok != PCL_OK) return ok;
    if (tracks_drape(crop)) return PCL_ERR_UNSUPPORTED;      // no curtains here: pcl_crop_tracking
  }
  int e = host_pipeline_ready(h);
  if (e != PCL_OK) return e;
  cudaStream_t s = (cudaStream_t)stream;
  // This step overwrites the device outputs: the D2H of this handle's previous
  // async step must have read them.  Other handles sharing `s` are not held up.
  if (h->pending_slot >= 0) PCL_CUDA(h, cudaStreamWaitEvent(s, h->ev_done[h->pending_slot], 0));
  e = step_host_enqueue(h, h_actions, d_actions, out, s);
  if (e != PCL_OK) return e;
  const uint8_t* d_view = out->d_board;
  size_t view_bytes = (size_t)h->batch * h->spec.rows * h->spec.pitch;
  if (crop) {                    // only the cropped view crosses PCIe
    // The same cropper attached to the handle (pcl_attach_cropper) has already run as
    // the step kernel's epilogue: nothing more to launch.
    const bool fused = h->base.has_cropper && h->base.cropper.out == d_crop &&
                       h->base.cropper.state == d_crop_state &&
                       memcmp(&h->base.cropper.crop, crop, sizeof(*crop)) == 0;
    e = fused ? PCL_OK : pcl_crop(h, crop, out->d_board, d_crop, d_crop_state, stream);
    if (e != PCL_OK) return e;
    d_view = d_crop;
    view_bytes = (size_t)h->batch * crop->rows * crop->cols;
  }
  PCL_CUDA(h, cudaEventRecord(h->ev_step[slot], s));
  PCL_CUDA(h, cudaStreamWaitEvent(h->copy_stream, h->ev_step[slot], 0));
  e = copy_outputs(h, out, d_view, view_bytes, h_view, h_reward, h_has_reward, h_discount, h_done,
                   h->copy_stream);
  if (e != PCL_OK) return e;
  PCL_CUDA(h, cudaEventRecord(h->ev_done[slot], h->copy_stream));
  h->pending_slot = slot;
  return PCL_OK;
}

int pcl_host_wait(pcl_handle* h, int slot) {
  if (!h || slot < 0 || slot >= PCL_HOST_SLOTS || !h->host_ready) return PCL_ERR_INVALID;
  PCL_CUDA(h, cudaEventSynchronize(h->ev_done[slot]));
  return PCL_OK;
}

int pcl_render(pcl_handle* h, const uint8_t* d_backdrop, int64_t backdrop_bstride,
               const uint8_t* d_curtains, const int32_t* d_sprites, const uint8_t* d_z_order,
               uint8_t* d_board, void* stream) {
  Range nvtx_range("pcl_render (Engine._render)");
  if (!h || !d_backdrop || !d_z_order || !d_board) return PCL_ERR_INVALID;
  if (h->spec.n_drapes > 0 && !d_curtains) return PCL_ERR_INVALID;
  if (h->spec.n_sprites > 0 && !d_sprites) return PCL_ERR_INVALID;
  pcl::RenderParams p;
  memset(&p, 0, sizeof(p));
  p.B = h->batch; p.H = h->spec.rows; p.W = h->spec.cols; p.pitch = h->spec.pitch;
  p.S = h->spec.n_sprites; p.D = h->spec.n_drapes;
  p.backdrop = d_backdrop; p.backdrop_bstride = backdrop_bstride;
  p.curtains = d_curtains; p.sprites = d_sprites; p.z_order = d_z_order; p.board = d_board;
  memcpy(p.sprite_char, h->spec.sprite_char, sizeof(p.sprite_char));
  memcpy(p.drape_char, h->spec.drape_char, sizeof(p.drape_char));
  return launched(h, pcl::launch_render(p, (cudaStream_t)stream), "launch_render");
}

namespace {
// Where drape d's curtain lives in the bound state: a window of a Scrolly pattern at
// the drape's corner, or bit rows of the board.  Fills d's fields of `p`.
int resolve_curtain(const pcl_handle* h, int d, pcl::LayersParams* p) {
  const pcl_spec& sp = h->spec;
  const pcl::CurtainAt at = h->program->curtain ? h->program->curtain(sp, d) : pcl::CurtainAt::kNone;
  if (at == pcl::CurtainAt::kPatternWindow || at == pcl::CurtainAt::kStaleWindow) {
    p->scrolly[d] = 1;
    p->bits[d] = h->st.d_pattern[d]; p->bits_bstride[d] = h->st.pattern_bstride[d];
    p->row_words[d] = sp.pattern_words;
    const bool coins = at == pcl::CurtainAt::kStaleWindow;
    p->stale_slot[d] = coins;
    // a pattern with a reset template is per env; the others are read-only, per level
    p->per_level[d] = !coins && h->st.d_level != nullptr && h->st.d_pattern_init[d] == nullptr;
  } else if (at == pcl::CurtainAt::kBits) {
    p->bits[d] = h->st.d_bits[d]; p->bits_bstride[d] = h->st.bits_bstride[d];
    p->row_words[d] = sp.bits_words;
  } else {
    return PCL_ERR_UNSUPPORTED;    // a curtain the layers kernel cannot read
  }
  return p->bits[d] ? PCL_OK : PCL_ERR_INVALID;
}

// A layers launch over `n_chars` planes; the caller fills the planes and resolves the
// drapes they read.
pcl::LayersParams layers_params(const pcl_handle* h, int n_chars, uint8_t* d_out) {
  const pcl_spec& sp = h->spec;
  pcl::LayersParams p;
  memset(&p, 0, sizeof(p));
  p.B = h->batch; p.H = sp.rows; p.W = sp.cols; p.pitch = sp.pitch;
  p.S = sp.n_sprites; p.D = sp.n_drapes; p.n_chars = n_chars;
  if (live_backdrop(sp)) {       // the Backdrop as its code left it, per env
    p.backdrop = h->backdrop_live; p.backdrop_bstride = (int64_t)sp.rows * sp.pitch;
    p.backdrop_per_env = 1;
  } else {
    p.backdrop = h->st.d_backdrop; p.backdrop_bstride = h->st.backdrop_bstride;
  }
  p.level = h->st.d_level; p.sprites = h->st.d_sprites; p.drapes = h->st.d_drapes;
  p.out = d_out;
  return p;
}
}  // namespace

int pcl_export_curtain(pcl_handle* h, int drape_index, uint8_t* d_out, void* stream) {
  if (!h || !d_out || drape_index < 0 || drape_index >= h->spec.n_drapes) return PCL_ERR_INVALID;
  if (!h->bound) return PCL_ERR_UNBOUND;
  pcl::LayersParams p = layers_params(h, 1, d_out);
  p.chars[0] = h->spec.drape_char[drape_index];
  p.sprite_of[0] = -1; p.drape_of[0] = (int8_t)drape_index;
  const int r = resolve_curtain(h, drape_index, &p);
  if (r != PCL_OK) return r;
  return launched(h, pcl::launch_layers(p, (cudaStream_t)stream), "launch_layers");
}

int pcl_layers(pcl_handle* h, const uint8_t* chars, int32_t n_chars, uint8_t* d_out,
               void* stream) {
  Range nvtx_range("pcl_layers");
  if (!h || !chars || !d_out || n_chars < 1 || n_chars > PCL_MAX_LAYER_CHARS)
    return PCL_ERR_INVALID;
  if (!h->bound) return PCL_ERR_UNBOUND;
  if (live_backdrop(h->spec) && !h->backdrop_live) return PCL_ERR_UNBOUND;
  const pcl_spec& sp = h->spec;
  pcl::LayersParams p = layers_params(h, n_chars, d_out);
  for (int d = 0; d < sp.n_drapes; ++d) {
    const int r = resolve_curtain(h, d, &p);
    if (r != PCL_OK) return r;
  }
  for (int k = 0; k < n_chars; ++k) {
    p.chars[k] = chars[k];
    p.sprite_of[k] = -1; p.drape_of[k] = -1;
    for (int s = 0; s < sp.n_sprites; ++s) if (sp.sprite_char[s] == chars[k]) p.sprite_of[k] = (int8_t)s;
    for (int d = 0; d < sp.n_drapes; ++d) if (sp.drape_char[d] == chars[k]) p.drape_of[k] = (int8_t)d;
  }
  return launched(h, pcl::launch_layers(p, (cudaStream_t)stream), "launch_layers");
}

namespace {
pcl::CropParams crop_params(const pcl_handle* h, const pcl_crop_spec* crop,
                            const uint8_t* d_board, uint8_t* d_crop, int32_t* d_crop_state) {
  pcl::CropParams p;
  memset(&p, 0, sizeof(p));
  p.B = h->batch; p.H = h->spec.rows; p.W = h->spec.cols; p.pitch = h->spec.pitch;
  p.S = h->spec.n_sprites; p.crop = *crop;
  p.sprites = h->st.d_sprites; p.plot = h->st.d_plot; p.board = d_board; p.out = d_crop;
  p.state = d_crop_state;
  // floor(2^32 / cols) + 1: __umulhi(i, recip) == i / cols for every i < 65536 (cols >= 1).
  p.cols_recip = crop->cols > 1 ? (uint32_t)(0x100000000ull / (uint32_t)crop->cols) + 1u : 0u;
  return p;
}
}  // namespace

int pcl_attach_cropper(pcl_handle* h, const pcl_crop_spec* crop, uint8_t* d_crop,
                       int32_t* d_crop_state) {
  if (!h) return PCL_ERR_INVALID;
  if (!h->bound) return PCL_ERR_UNBOUND;
  if (!crop) {                                               // detach
    h->base.has_cropper = 0;
    return PCL_OK;
  }
  if (!d_crop) return PCL_ERR_INVALID;
  if (!h->program->crop_epilogue) return PCL_ERR_UNSUPPORTED;
  const int ok = crop_spec_ok(h, crop);
  if (ok != PCL_OK) return ok;
  if (tracks_drape(crop)) return PCL_ERR_UNSUPPORTED;        // drape medians need scratch memory
  h->base.cropper = crop_params(h, crop, nullptr, d_crop, d_crop_state);
  h->base.has_cropper = 1;
  return PCL_OK;
}

int pcl_crop(pcl_handle* h, const pcl_crop_spec* crop, const uint8_t* d_board, uint8_t* d_crop,
             int32_t* d_crop_state, void* stream) {
  return pcl_crop_tracking(h, crop, d_board, d_crop, d_crop_state, nullptr, stream);
}

int pcl_crop_tracking(pcl_handle* h, const pcl_crop_spec* crop, const uint8_t* d_board,
                      uint8_t* d_crop, int32_t* d_crop_state,
                      const uint8_t* const* d_curtains, void* stream) {
  Range nvtx_range("pcl_crop (ScrollingCropper.crop)");
  if (!h || !crop || !d_board || !d_crop) return PCL_ERR_INVALID;
  if (!h->bound) return PCL_ERR_UNBOUND;
  const int ok = crop_spec_ok(h, crop);
  if (ok != PCL_OK) return ok;
  pcl::CropParams p = crop_params(h, crop, d_board, d_crop, d_crop_state);
  for (int i = 0; i < PCL_MAX_TRACK && crop->track[i] != 0; ++i) {
    if (crop->track[i] > 0) continue;
    if (!d_curtains || !d_curtains[i]) return PCL_ERR_INVALID;
    if (h->spec.rows > 128 || h->spec.cols > 128) return PCL_ERR_UNSUPPORTED;
    p.curtains[i] = d_curtains[i];
  }
  return launched(h, pcl::launch_crop(p, (cudaStream_t)stream), "launch_crop");
}

int pcl_crop_handoff(pcl_handle* h, const pcl_crop_spec* crop, const uint8_t* d_board,
                     int32_t* d_crop_state, const pcl_outputs* out, const pcl_handoff* x,
                     void* stream) {
  Range nvtx_range("pcl_crop_handoff");
  if (!h || !crop || !d_board || !out || !x) return PCL_ERR_INVALID;
  if (!h->bound) return PCL_ERR_UNBOUND;
  if (!outputs_set(*out)) return PCL_ERR_INVALID;
  if (float_rewards(h)) return PCL_ERR_UNSUPPORTED;     // the record's reward is int32
  const int ok = crop_spec_ok(h, crop);
  if (ok != PCL_OK) return ok;
  if (tracks_drape(crop)) return PCL_ERR_UNSUPPORTED;        // drape tracking: pcl_crop_tracking
  const int view = crop->rows * crop->cols;
  if (x->n_peers < 1 || x->n_peers > PCL_MAX_PEERS || x->rank < 0 || x->rank >= x->n_peers)
    return PCL_ERR_INVALID;
  if ((x->record_bytes & 15) || x->record_bytes < PCL_HANDOFF_RECORD_BYTES(view) ||
      x->record_bytes > 256) return PCL_ERR_INVALID;
  if (!x->d_local || x->first_row < 0 || x->first_row + h->batch > x->rows) return PCL_ERR_INVALID;
  const pcl::CropParams p = crop_params(h, crop, d_board, nullptr, d_crop_state);
  pcl::HandoffParams q;
  memset(&q, 0, sizeof(q));
  q.n_peers = x->n_peers; q.rank = x->rank; q.record_bytes = x->record_bytes;
  q.rows = x->rows; q.first_row = x->first_row;
  for (int i = 0; i < x->n_peers; ++i) {
    if (!x->d_peer_base[i] || !x->d_peer_flags[i]) return PCL_ERR_INVALID;
    q.peer_base[i] = x->d_peer_base[i]; q.peer_flags[i] = x->d_peer_flags[i];
  }
  q.multicast = x->d_multicast; q.local = x->d_local; q.out = *out;
  q.n_bufs = x->n_bufs == 0 ? 2 : x->n_bufs;
  if (x->mode & ~(PCL_HANDOFF_LAG | PCL_HANDOFF_SIGNAL_KERNEL)) return PCL_ERR_INVALID;
  q.lag = (x->mode & PCL_HANDOFF_LAG) ? 1 : 0;
  q.signal_kernel = (x->mode & PCL_HANDOFF_SIGNAL_KERNEL) ? 1 : 0;
  if (q.n_bufs < 2 || q.n_bufs > 8 || (q.lag == 1 && q.n_bufs < 3)) return PCL_ERR_INVALID;
  const int r = launched(h, pcl::launch_crop_handoff(p, q, (cudaStream_t)stream), "launch_crop_handoff");
  if (r == PCL_OK && q.signal_kernel) h->launches += 1;      // the one-warp publish kernel
  return r;
}

int pcl_pack_handoff(pcl_handle* h, const uint8_t* d_view, int32_t view_bytes,
                     const pcl_outputs* out, uint8_t* d_packed, void* stream) {
  if (!h || !d_view || !out || !d_packed || view_bytes <= 0) return PCL_ERR_INVALID;
  if (!outputs_set(*out)) return PCL_ERR_INVALID;
  if (float_rewards(h)) return PCL_ERR_UNSUPPORTED;     // the record's reward is int32
  pcl::PackParams p;
  memset(&p, 0, sizeof(p));
  p.B = h->batch; p.view_bytes = view_bytes;
  p.record_bytes = PCL_HANDOFF_RECORD_BYTES(view_bytes);
  p.view = d_view; p.out = *out; p.packed = d_packed;
  return launched(h, pcl::launch_pack_handoff(p, (cudaStream_t)stream), "launch_pack_handoff");
}

int pcl_pack_handoff_peers(pcl_handle* h, const uint8_t* d_view, int32_t view_bytes,
                           const pcl_outputs* out, uint8_t* const* d_peer_bases,
                           int32_t n_peers, int64_t first_row, void* stream) {
  if (!h || !d_view || !out || !d_peer_bases || view_bytes <= 0 || first_row < 0)
    return PCL_ERR_INVALID;
  if (n_peers < 1 || n_peers > PCL_MAX_PEERS) return PCL_ERR_INVALID;
  if (!outputs_set(*out)) return PCL_ERR_INVALID;
  if (float_rewards(h)) return PCL_ERR_UNSUPPORTED;     // the record's reward is int32
  pcl::PackParams p;
  memset(&p, 0, sizeof(p));
  p.B = h->batch; p.view_bytes = view_bytes;
  p.record_bytes = PCL_HANDOFF_RECORD_BYTES(view_bytes);
  p.view = d_view; p.out = *out;
  p.n_peers = n_peers; p.first_row = first_row;
  for (int i = 0; i < n_peers; ++i) {
    if (!d_peer_bases[i]) return PCL_ERR_INVALID;
    p.peers[i] = d_peer_bases[i];
  }
  return launched(h, pcl::launch_pack_handoff(p, (cudaStream_t)stream), "launch_pack_handoff");
}

int pcl_observe(pcl_handle* h, const pcl_observe_spec* spec, const void* d_table,
                const uint8_t* d_valid, const uint8_t* d_board, void* d_out,
                int32_t* d_unknown, void* stream) {
  Range nvtx_range("pcl_observe");
  if (!h || !spec || !d_table || !d_board || !d_out) return PCL_ERR_INVALID;
  if (spec->depth < 1 || spec->depth > 32 || spec->dtype < 0 || spec->dtype > 5)
    return PCL_ERR_INVALID;
  pcl::ObserveParams p;
  memset(&p, 0, sizeof(p));
  p.B = h->batch; p.H = h->spec.rows; p.W = h->spec.cols; p.pitch = h->spec.pitch;
  p.depth = spec->depth; p.dtype = spec->dtype;
  p.words = spec->dtype >= 3 ? 2 : 1;     // 8-byte elements: two u32; 2-byte: two u8
  p.stride_b = spec->stride_b * p.words; p.stride_d = spec->stride_d * p.words;
  p.stride_r = spec->stride_r * p.words; p.stride_c = spec->stride_c * p.words;
  p.table = d_table; p.valid = d_valid; p.board = d_board; p.out = d_out;
  p.unknown = d_unknown;
  return launched(h, pcl::launch_observe(p, (cudaStream_t)stream), "launch_observe");
}

int pcl_error_codes(pcl_handle* h, int32_t* d_out, void* stream) {
  if (!h || !d_out) return PCL_ERR_INVALID;
  if (!h->bound) return PCL_ERR_UNBOUND;
  gather_errors<<<(h->batch + 255) / 256, 256, 0, (cudaStream_t)stream>>>(h->st.d_plot, d_out,
                                                                           h->batch);
  return launched(h, cudaGetLastError(), "gather_errors");
}

int pcl_launch_count(pcl_handle* h, int64_t* out) {
  if (!h || !out) return PCL_ERR_INVALID;
  *out = h->launches;
  return PCL_OK;
}

}  // extern "C"
