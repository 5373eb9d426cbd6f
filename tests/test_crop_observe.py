"""Croppers feeding the post-processors, without a GPU.

- The oracle composition (`crop_window` / `ScrollingCrop`, then the oracle's
  post-processors) against the reference's own croppers and post-processors, frozen in
  tests/golden/windowobs_*.npz: outputs, and which calls raised RuntimeError.
- C-boundary refusals of `pcl_crop_observe` on a handle that reaches no device (device
  -1, made-up addresses): each is refused before anything is enqueued.
- What ptxas made of the kernel in the built libpcl.so: no local-memory stack.
"""

import ctypes as C

import numpy as np
import pytest

import boundary_sweep
import crop_cases as cc
import crop_observe_cases as coc
from pycolab_b200 import _lib
from test_kernel_resources import _cuobjdump, _resource_usage


@pytest.mark.parametrize('name', coc.golden_names())
def test_oracle_composition_matches_the_reference_goldens(name):
  c, seq, want, outs = coc.load_golden(name)
  assert len(outs) == len(c['croppers']) * len(coc.PROCESSORS)
  for k, cropper in enumerate(c['croppers']):
    got = cc.oracle(c, cropper, seq, with_layers=True)
    for proc in coc.PROCESSORS:
      ref_out, ref_raised = outs[(k, proc['name'])]
      for t, (crops, corners, lays) in enumerate(got):
        msg = '%s cropper %d %s t=%d' % (name, k, proc['name'], t)
        out, raised = coc.oracle_apply(proc, crops, lays)
        assert raised == bool(ref_raised[t].any()), msg
        assert out.dtype == ref_out.dtype and out.shape == ref_out[t].shape, msg
        np.testing.assert_array_equal(out, ref_out[t], err_msg=msg)


def test_goldens_cover_what_they_promise():
  """Every processor raises somewhere and not everywhere where its mapping lacks a
  character; windows past the board and un-occluded layers that differ from the
  cropped board's are in the goldens."""
  raised, off_board, unoccluded = {}, 0, 0
  for name in coc.golden_names():
    c, seq, want, outs = coc.load_golden(name)
    for (k, p), (_, r) in outs.items():
      raised.setdefault(p, []).append(r.reshape(-1))
    for k, cropper in enumerate(c['croppers']):
      for crops, corners, lays in want[k]:
        rows, cols = cropper['rows'], cropper['cols']
        off_board += int(((corners < 0).any(1) | (corners[:, 0] + rows > c['H']) |
                          (corners[:, 1] + cols > c['W'])).sum())
        unoccluded += sum(int((lay[ch] != (crops[e] == ord(ch))).any())
                          for e, lay in enumerate(lays) for ch in lay)
  for p, flags in raised.items():
    flags = np.concatenate(flags)
    lacks = coc.BY_NAME[p]['kind'] == 'array' and set(coc.ALL) - set(coc.BY_NAME[p]['mapping'])
    assert (0 < flags.sum() < len(flags)) if lacks else not flags.any(), p
  assert off_board > 0 and unoccluded > 0
  assert set(n for n, _, _ in coc.GOLDEN_CASES) >= {'b8x14_fixed', 'b32x32_two_croppers'}


# ---- C boundary --------------------------------------------------------------------

FAKE = boundary_sweep.FAKE


def _none_handle(H=16, W=16):
  lib = _lib.load()
  spec = _lib.Spec()
  spec.abi_version, spec.program = _lib.ABI_VERSION, _lib.PROG_NONE
  spec.rows, spec.cols, spec.pitch = H, W, cc.pitch(W)
  spec.n_sprites, spec.n_drapes = 2, 2
  h = C.c_void_p()
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(h)) == _lib.OK
  assert lib.pcl_bind_state(h, C.byref(boundary_sweep._full_state())) == _lib.OK
  return lib, h


def _crop_spec(rows=5, cols=7, track=None, pad='.'):
  from pycolab_b200 import batched
  return batched.scrolling_crop_spec(rows, cols, 0, pad_char=pad, scroll_margins=(0, 0),
                                     track=track)


def _call(lib, h, crop=None, board=FAKE, curtains=None, depth=3, dtype=2, table=FAKE,
          out=FAKE, planes=None, plane_of=None):
  crop = _crop_spec() if crop is None else crop
  spec = _lib.ObserveSpec(depth, dtype, 3 * 35, 35, 7, 1)
  return lib.pcl_crop_observe(h, C.byref(crop), board, FAKE, curtains, C.byref(spec), table,
                              None, planes, plane_of, -1, 0, 0, 0, out, None, None)


def test_refuses_nulls_depths_and_dtypes():
  lib, h = _none_handle()
  try:
    assert _call(lib, h, board=None) == _lib.ERR_INVALID
    assert _call(lib, h, table=None) == _lib.ERR_INVALID
    assert _call(lib, h, out=None) == _lib.ERR_INVALID
    assert _call(lib, h, board=None, planes=FAKE) == _lib.ERR_INVALID   # no plane map
    assert lib.pcl_crop_observe(h, None, FAKE, FAKE, None,
                                C.byref(_lib.ObserveSpec(1, 0, 1, 1, 1, 1)), FAKE, None, None,
                                None, -1, 0, 0, 0, FAKE, None, None) == _lib.ERR_INVALID
    assert lib.pcl_crop_observe(h, C.byref(_crop_spec()), FAKE, FAKE, None, None, FAKE, None,
                                None, None, -1, 0, 0, 0, FAKE, None, None) == _lib.ERR_INVALID
    assert lib.pcl_crop_observe(None, C.byref(_crop_spec()), FAKE, FAKE, None,
                                C.byref(_lib.ObserveSpec(1, 0, 1, 1, 1, 1)), FAKE, None, None,
                                None, -1, 0, 0, 0, FAKE, None, None) == _lib.ERR_INVALID
    for depth in (0, -1):
      assert _call(lib, h, depth=depth) == _lib.ERR_INVALID
    for dtype in (-1, 6, 99):
      assert _call(lib, h, dtype=dtype) == _lib.ERR_INVALID
    assert _call(lib, h, crop=_crop_spec(4, 6, [3])) == _lib.ERR_INVALID      # no sprite 2
    assert _call(lib, h, crop=_crop_spec(20, 20, pad=None)) == _lib.ERR_INVALID   # past the board
  finally:
    lib.pcl_destroy(h)


@pytest.mark.parametrize('window', [(256, 256), (65536, 1), (1, 65536), (300, 300)], ids=str)
def test_windows_past_the_cell_limit_are_unsupported(window):
  lib, h = _none_handle()
  try:
    for track in (None, [1], [-1, 2]):
      curtains = (C.c_void_p * _lib.MAX_TRACK)(*([FAKE] * _lib.MAX_TRACK))
      assert _call(lib, h, _crop_spec(window[0], window[1], track),
                   curtains=curtains) == _lib.ERR_UNSUPPORTED, track
  finally:
    lib.pcl_destroy(h)


@pytest.mark.parametrize('track', [[-1], [1, -2], [-2, 1, -1]], ids=str)
def test_drape_tracking_needs_curtains(track):
  """A tracking list naming a drape needs that drape's curtain (INVALID without), and a
  board of at most 128 x 128 (UNSUPPORTED past it)."""
  lib, h = _none_handle()
  try:
    assert _call(lib, h, _crop_spec(5, 7, track)) == _lib.ERR_INVALID
    partial = (C.c_void_p * _lib.MAX_TRACK)()
    assert _call(lib, h, _crop_spec(5, 7, track), curtains=partial) == _lib.ERR_INVALID
  finally:
    lib.pcl_destroy(h)
  lib, h = _none_handle(129, 8)
  try:
    curtains = (C.c_void_p * _lib.MAX_TRACK)(*([FAKE] * _lib.MAX_TRACK))
    assert _call(lib, h, _crop_spec(5, 7, track), curtains=curtains) == _lib.ERR_UNSUPPORTED
  finally:
    lib.pcl_destroy(h)


def test_refuses_an_unbound_handle():
  lib = _lib.load()
  spec = _lib.Spec()
  spec.abi_version, spec.program = _lib.ABI_VERSION, _lib.PROG_NONE
  spec.rows, spec.cols, spec.pitch, spec.n_sprites = 16, 16, 16, 2
  h = C.c_void_p()
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(h)) == _lib.OK
  try:
    assert _call(lib, h) == _lib.ERR_UNBOUND
  finally:
    lib.pcl_destroy(h)


@pytest.mark.skipif(_cuobjdump() is None, reason='cuobjdump not found')
def test_kernel_has_no_local_memory_stack():
  import os
  assert os.path.exists(_lib.LIB_PATH), 'build libpcl.so first'
  kernels = {n: u for n, u in _resource_usage(_lib.LIB_PATH).items()
             if 'crop_observe_kernel' in n}
  assert len(kernels) == 2, kernels               # 1- / 2-byte and 4- / 8-byte elements
  for name, u in kernels.items():
    assert u['STACK'] == 0, (name, u)
