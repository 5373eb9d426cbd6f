// pcl_crop.cuh — the cropper's device functions (cropping.py:118-598), shared by the
// stand-alone crop kernels (render.cu) and by step kernels that run an ATTACHED cropper
// as their epilogue (pcl_attach_cropper).  Warp-wide: every lane of an env's warp calls
// them together.
#pragma once

#include "pcl_device.cuh"
#include "pcl_kernels.cuh"

namespace pcl {

// (median row, median column) of a byte curtain's cells, as `_centroid` computes
// them for a Drape (cropping.py:583-596: np.median of the nonzero coordinates,
// truncated).  Warp-wide; `hist` is this warp's 256-int scratch.  false = empty.
__device__ __forceinline__ bool curtain_centroid(const uint8_t* curtain, int H, int W, int pitch, int lane,
                                 int* hist, int* crow, int* ccol) {
  int* rows = hist;
  int* cols = hist + 128;
  int n = 0;
  for (int c = lane; c < 128; c += 32) cols[c] = 0;
  __syncwarp();
  for (int r = 0; r < H; ++r) {
    int in_row = 0;
    for (int c0 = 0; c0 < W; c0 += 32) {
      const int c = c0 + lane;
      const bool on = c < W && curtain[(int64_t)r * pitch + c] != 0;
      in_row += __popc(__ballot_sync(0xffffffffu, on));
      if (on) cols[c] += 1;                  // lane `c & 31` owns column c
    }
    if (lane == 0) rows[r] = in_row;
    n += in_row;
  }
  __syncwarp();
  if (n == 0) return false;
  // k-th smallest coordinate from the histograms; the median of an even count is
  // the mean of the two middle values, truncated (int(np.median(...))).
  auto kth = [&](const int* h, int len, int k) {
    int seen = 0;
    for (int i = 0; i < len; ++i) { seen += h[i]; if (seen > k) return i; }
    return len - 1;
  };
  const int k1 = (n - 1) / 2, k2 = n / 2;
  *crow = (kth(rows, H, k1) + kth(rows, H, k2)) / 2;
  *ccol = (kth(cols, W, k1) + kth(cols, W, k2)) / 2;
  return true;
}

// ScrollingCropper.crop (cropping.py:393-426) up to the window corner: follow the
// first visible entity of the tracking list, pan / saccade, persist the corner.
// Warp-wide; returns the corner every lane must use for _do_crop.
__device__ __forceinline__ void crop_corner(const CropParams& p, int env, int lane, int* hist,
                                            int* out_wr, int* out_wc) {
  const pcl_crop_spec& c = p.crop;
  int32_t* plot = p.plot + (int64_t)env * PCL_PLOT_WORDS;
  const bool fixed = c.sprite_index < 0;                  // FixedCropper :229-310
  bool have = false;                                      // _centroid :544-598
  int crow = 0, ccol = 0;
  if (!fixed) {
#pragma unroll
    for (int e = 0; e < PCL_MAX_TRACK && !have; ++e) {
      const int code = c.track[0] == 0 ? (e == 0 ? c.sprite_index + 1 : 0) : c.track[e];
      if (code == 0) break;
      if (code > 0) {
        const int32_t* rec = p.sprites + ((int64_t)env * p.S + code - 1) * PCL_SPRITE_WORDS;
        if (rec[PCL_S_FLAGS] & 1) { have = true; crow = rec[PCL_S_ROW]; ccol = rec[PCL_S_COL]; }
      } else {
        have = curtain_centroid(p.curtains[e] + (int64_t)env * p.H * p.pitch, p.H, p.W, p.pitch,
                                lane, hist, &crow, &ccol);
      }
    }
  }
  // Corner state: the caller's per-cropper array, or the plot record's one slot.
  int32_t* state = p.state ? p.state + (int64_t)env * 4 : plot + PCL_P_CROP_R;
  const int episode = plot[PCL_P_EPISODES];
  int wr = fixed ? c.offset_rows : state[0];
  int wc = fixed ? c.offset_cols : state[1];
  // A new episode is a new Engine upstream: set_engine() forgets the corner.
  const int init = fixed ? 1 : (p.state ? (state[2] && state[3] == episode) : state[2]);
  const bool pad = c.pad_char >= 0;
  auto rectify = [&]() {                                  // :533-542
    wr = max(0, wr) - max(0, wr + c.rows - p.H);
    wc = max(0, wc) - max(0, wc + c.cols - p.W);
  };
  auto initialise = [&](int orow, int ocol) {             // :438-458
    if (!have) { wr = 0; wc = 0; return; }
    wr = crow - orow; wc = ccol - ocol;
    if (!pad) rectify();
  };
  if (!init) {
    initialise(c.rows / 2 + c.offset_rows, c.cols / 2 + c.offset_cols);
  } else if (have) {
    const int mr = c.margin_rows, mc = c.margin_cols;
    bool can_v = (mr - 1 <= crow - wr) && (crow - wr <= c.rows - mr);   // :460-505
    bool can_h = (mc - 1 <= ccol - wc) && (ccol - wc <= c.cols - mc);
    if (!pad) {
      if (!can_v) {
        if (wr <= 0) can_v = crow <= mr;
        else if (wr >= p.H - c.rows) can_v = crow >= wr + c.rows - mr;
      } else if (!can_h) {
        if (wc <= 0) can_h = ccol <= mc;
        else if (wc >= p.W - c.cols) can_h = ccol >= wc + c.cols - mc;
      }
    }
    if (can_v && can_h) {                                 // _pan_to :507-531
      int dr = min(0, crow - wr - mr);
      int dc = min(0, ccol - wc - mc);
      if (dr == 0) dr += max(0, crow - wr - c.rows + mr + 1);
      if (dc == 0) dc += max(0, ccol - wc - c.cols + mc + 1);
      wr += dr; wc += dc;
      if (!pad) rectify();
    } else if (c.saccade) {
      initialise(c.rows / 2, c.cols / 2);
    }
  }
  __syncwarp();
  if (lane == 0 && !fixed) {
    state[0] = wr; state[1] = wc; state[2] = 1;
    if (p.state) state[3] = episode;
  }
  *out_wr = wr; *out_wc = wc;
}

// Cell (jr, jc) of the window at corner (wr, wc) of a plane with `pitch` bytes per row:
// the plane's byte on the board, `padv` outside it (_do_crop :118-227).
__device__ __forceinline__ uint32_t crop_cell(const CropParams& p, const uint8_t* plane,
                                              int64_t pitch, int wr, int wc, int jr, int jc,
                                              uint32_t padv) {
  const int r = wr + jr, cc2 = wc + jc;
  uint32_t b = padv;
  if ((unsigned)r < (unsigned)p.H && (unsigned)cc2 < (unsigned)p.W)
    b = plane[(int64_t)r * pitch + cc2];
  return b;
}

// Four consecutive cells i .. i + 3 of the crop window (row-major over rows x cols)
// as one little-endian word, pad character outside the board (_do_crop :118-227).
// One division per word (by a runtime width, as a multiply-high with the reciprocal in
// CropParams::cols_recip: exact for i < 65536), then the cell walks along the row.
__device__ __forceinline__ uint32_t crop_word(const CropParams& p, const uint8_t* board, int wr,
                                              int wc, int i, int cells) {
  const pcl_crop_spec& c = p.crop;
  const uint32_t padv = c.pad_char >= 0 ? (uint32_t)c.pad_char : 0u;
  int jr = c.cols == 1 ? i : (int)__umulhi((uint32_t)i, p.cols_recip);   // i / cols
  int jc = i - jr * c.cols;                                // i % cols
  uint32_t v = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (i + k >= cells) break;
    v |= crop_cell(p, board, p.pitch, wr, wc, jr, jc, padv) << (8 * k);
    if (++jc == c.cols) { jc = 0; ++jr; }
  }
  return v;
}


// An attached cropper as the last act of a step kernel (pcl_attach_cropper): the warp that
// has just stored its env's records and board crops that board into `a.out`.  The caller
// has synchronised the warp after those stores (they are this warp's own, so the loads
// below see them); scratch for drape medians is not available here, so the launcher
// refuses tracking lists that name drapes.
// `rec_sprites` / `rec_plot`: the env's sprite and plot records where the calling warp
// still holds them (shared memory), or NULL to read them back from global memory.
__device__ __forceinline__ void crop_epilogue(const CropParams& a, const uint8_t* d_board,
                                              int env, int lane,
                                              const int32_t* rec_sprites = nullptr,
                                              int32_t* rec_plot = nullptr) {
  CropParams c = a;
  c.board = d_board;
  // crop_corner indexes sprites / plot by env: bias the warp-local copies so that the
  // env-th record IS the local one.  The plot's own corner slot (state == NULL) must stay
  // in global memory, so the local plot is only used with a caller-owned state array.
  if (rec_sprites) c.sprites = rec_sprites - (int64_t)env * c.S * PCL_SPRITE_WORDS;
  if (rec_plot && c.state) c.plot = rec_plot - (int64_t)env * PCL_PLOT_WORDS;
  int wr, wc;
  crop_corner(c, env, lane, nullptr, &wr, &wc);
  const uint8_t* board = d_board + (int64_t)env * c.H * c.pitch;
  const int cells = c.crop.rows * c.crop.cols;
  uint8_t* out = c.out + (int64_t)env * cells;
  const int mis = (int)(reinterpret_cast<uintptr_t>(out) & 3);
  const int head = mis ? 4 - mis : 0;
  if (lane < head && lane < cells) out[lane] = (uint8_t)crop_word(c, board, wr, wc, lane, cells);
  for (int i = head + lane * 4; i < cells; i += 128) {
    const uint32_t v = crop_word(c, board, wr, wc, i, cells);
    if (i + 4 <= cells) {
      *reinterpret_cast<uint32_t*>(out + i) = v;
    } else {
      for (int k = 0; i + k < cells; ++k) out[i + k] = (uint8_t)(v >> (8 * k));
    }
  }
}

}  // namespace pcl
