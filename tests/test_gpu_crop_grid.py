"""The croppers on the device against the oracle, byte for byte, over `crop_cases.CASES`.

- Direct: a no-program handle bound to device sprite and plot records that the test
  writes each frame; `pcl_crop` / `pcl_crop_tracking` write every env's view into the
  middle of a sentinel-filled allocation at byte offsets 0..3 (so each env's row starts
  at every alignment); the guard bytes must come back untouched, and the corner state
  (the caller's array or the plot record's slot) must hold the oracle's corner.
- Fused hand-off: `pcl_crop_handoff` on one rank, records of more than the minimum size:
  view bytes, zero padding, reward / discount / done words, alternating parts.
- Attached epilogue: scrolly_maze's attached cropper against the stand-alone kernel.
- Facade: `ScrollingCropper` / `FixedCropper` with occlusion_in_layers=False (every
  cropped layer), tracking a box_world key, windows past PCL_MAX_CROP_CELLS.
- `play_host_async` with a spec it refuses: nothing is stepped or enqueued.
"""

import ctypes as C

import numpy as np
import pytest

import crop_cases as cc
from oracle import engine_model as em
from oracle import games as ogames

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5
GUARD = 64


class _Direct(object):
  """A PROG_NONE handle of a case's shape with device records the test writes."""

  def __init__(self, c):
    import torch
    from pycolab_b200 import _lib
    self.lib = lib = _lib.load()
    self.c = c
    B, H, W, S, D = c['B'], c['H'], c['W'], c['S'], c['D']
    spec = _lib.Spec()
    spec.abi_version, spec.program = _lib.ABI_VERSION, _lib.PROG_NONE
    spec.rows, spec.cols, spec.pitch = H, W, cc.pitch(W)
    spec.n_sprites, spec.n_drapes = S, D
    self.h = C.c_void_p()
    _lib.check(lib.pcl_create(C.byref(spec), B, 0, C.byref(self.h)), 'pcl_create')
    i32 = dict(dtype=torch.int32, device='cuda')
    self.sprites = torch.zeros((B, max(S, 1), _lib.SPRITE_WORDS), **i32)
    self.drapes = torch.zeros((B, max(D, 1), _lib.DRAPE_WORDS), **i32)
    self.plot = torch.zeros((B, _lib.PLOT_WORDS), **i32)
    self.backdrop = torch.zeros((1, H, cc.pitch(W)), dtype=torch.uint8, device='cuda')
    self.boards = torch.zeros((B, H, cc.pitch(W)), dtype=torch.uint8, device='cuda')
    self.curtains = torch.zeros((max(D, 1), B, H, cc.pitch(W)), dtype=torch.uint8,
                                device='cuda')
    st = _lib.State()
    st.d_backdrop = self.backdrop.data_ptr()
    st.d_sprites = st.d_sprites_init = self.sprites.data_ptr()
    st.d_drapes = st.d_drapes_init = self.drapes.data_ptr()
    st.d_plot = st.d_plot_init = self.plot.data_ptr()
    _lib.check(lib.pcl_bind_state(self.h, C.byref(st)), 'pcl_bind_state')

  def show(self, f):
    import torch
    from pycolab_b200 import _lib
    c = self.c
    self.boards.copy_(torch.from_numpy(f.boards))
    rec = np.zeros(tuple(self.sprites.shape), np.int32)
    rec[:, :c['S'], _lib.S_ROW] = f.sprites[..., 0]
    rec[:, :c['S'], _lib.S_COL] = f.sprites[..., 1]
    rec[:, :c['S'], _lib.S_FLAGS] = f.sprites[..., 2]
    self.sprites.copy_(torch.from_numpy(rec))
    # A restart rebuilds the plot record from its template, which clears the built-in
    # cropper slot (state NULL); the episode counter moves on.
    moved = torch.from_numpy(f.episode).cuda() != self.plot[:, _lib.P_EPISODES]
    self.plot[moved, _lib.P_CROP_R:_lib.P_CROP_INIT + 1] = 0
    self.plot[:, _lib.P_EPISODES] = torch.from_numpy(f.episode).cuda()
    if c['D']:
      cur = np.zeros(tuple(self.curtains.shape), np.uint8)
      cur[:, :, :, :c['W']] = f.curtains.transpose(1, 0, 2, 3)
      self.curtains.copy_(torch.from_numpy(cur))

  def crop(self, spec, state, out_ptr):
    from pycolab_b200 import _lib
    stream = C.c_void_p(__import__('torch').cuda.current_stream().cuda_stream)
    state_ptr = None if state is None else state.data_ptr()
    if any(code < 0 for code in spec.track):
      ptrs = (C.c_void_p * _lib.MAX_TRACK)()
      for i, code in enumerate(spec.track):
        if code < 0:
          ptrs[i] = self.curtains[-code - 1].data_ptr()
      return self.lib.pcl_crop_tracking(self.h, C.byref(spec), self.boards.data_ptr(), out_ptr,
                                        state_ptr, ptrs, stream)
    return self.lib.pcl_crop(self.h, C.byref(spec), self.boards.data_ptr(), out_ptr, state_ptr,
                             stream)

  def close(self):
    self.lib.pcl_destroy(self.h)


@pytest.mark.parametrize('name', [c['name'] for c in cc.CASES])
def test_direct_grid(name):
  c = cc.BY_NAME[name]
  seq = cc.frames(c)
  _direct(c, seq, [cc.oracle(c, k, seq) for k in c['croppers']])


@pytest.mark.parametrize('name', cc.golden_names())
def test_direct_reference_goldens(name):
  """The reference's own crops (tests/golden/cropgrid_*.npz) replayed through the same
  path; each layer of the observation cut at the device's corner (checked equal to the
  reference's) as the facade cuts it
  (`cropping.crop_layers`) is the reference's cropped layer."""
  c, seq, want = cc.load_golden(name)
  _direct(c, seq, want)


def _direct(c, seq, wants):
  """Run every cropper of case `c` over `seq` through pcl_crop / pcl_crop_tracking and
  require wants[k][t] = (crops, corners[, layer dicts]) of cropper k at frame t."""
  import torch
  from pycolab_b200 import _lib, cropping
  name, B = c['name'], c['B']
  specs = [cc.crop_spec(c, k) for k in c['croppers']]
  states = [torch.zeros((B, 4), dtype=torch.int32, device='cuda') if k['state'] == 'own'
            else None for k in c['croppers']]
  dev = _Direct(c)
  try:
    for t, f in enumerate(seq):
      dev.show(f)
      for k, cropper in enumerate(c['croppers']):
        cells = cropper['rows'] * cropper['cols']
        off = (t + k) % 4
        buf = torch.full((2 * GUARD + B * cells + 4,), SENTINEL, dtype=torch.uint8,
                         device='cuda')
        _lib.check(dev.crop(specs[k], states[k], buf.data_ptr() + GUARD + off), 'crop')
        torch.cuda.synchronize()
        raw = buf.cpu().numpy()
        msg = '%s cropper %d t=%d offset %d' % (name, k, t, off)
        assert (raw[:GUARD + off] == SENTINEL).all(), msg + ': head guard written'
        assert (raw[GUARD + off + B * cells:] == SENTINEL).all(), msg + ': tail guard written'
        got = raw[GUARD + off:GUARD + off + B * cells].reshape(B, cropper['rows'],
                                                              cropper['cols'])
        want, corners = wants[k][t][:2]
        bad = np.nonzero((got != want).reshape(B, -1).any(1))[0]
        assert not len(bad), '%s: envs %s differ (first: got\n%s\nwant\n%s)' % (
            msg, bad[:8].tolist(), got[bad[0]], want[bad[0]])
        if cropper['kind'] == 'scroll':
          if states[k] is not None:
            st = states[k].cpu().numpy()
            np.testing.assert_array_equal(st[:, :2], corners, err_msg=msg + ' corner')
            np.testing.assert_array_equal(st[:, 3], f.episode, err_msg=msg + ' episode')
          else:
            slot = dev.plot[:, _lib.P_CROP_R:_lib.P_CROP_C + 1].cpu().numpy()
            np.testing.assert_array_equal(slot, corners, err_msg=msg + ' plot corner')
        if len(wants[k][t]) > 2:
          pad = cc.pad_char(c, cropper)
          for e in range(B):
            got_layers = cropping.crop_layers(cc.layers(c, f, e), tuple(corners[e]),
                                              cropper['rows'], cropper['cols'], pad)
            for ch, plane in wants[k][t][2][e].items():
              np.testing.assert_array_equal(got_layers[ch], plane,
                                            err_msg='%s env %d layer %r' % (msg, e, ch))
  finally:
    dev.close()


@pytest.mark.parametrize('name', ['b1x1_w1x1', 'b37x1_w1x5_pad', 'b5x7_w3x5_b4099',
                                  'b8x14_w4x6', 'b33x65_w9x9', 'b64x64_w4x6_b1',
                                  'b8x14_fixed'])
def test_fused_handoff_single_rank(name):
  """pcl_crop_handoff, one rank, signalling in the kernel: each env's record in this
  step's part is its oracle view, zero padding, then reward, discount and done |
  has_reward << 8, zeros up to record_bytes (here 16 or 32 bytes past the minimum); the
  other part is untouched."""
  import torch
  from pycolab_b200 import _lib
  from test_dist import pack_records
  c = cc.BY_NAME[name]
  B = c['B']
  seq = cc.frames(c)
  dev = _Direct(c)
  rs = np.random.RandomState(3)
  try:
    for k, cropper in enumerate(c['croppers']):
      if cropper['kind'] == 'scroll':                # the hand-off tracks sprites only
        cropper = dict(cropper, track=[n for n in cropper['track'] if n[0] == 's'] or ['s0'])
      spec = cc.crop_spec(c, cropper)
      want = cc.oracle(c, cropper, seq)
      view = cropper['rows'] * cropper['cols']
      least = ((view + 3) // 4 * 4 + 12 + 15) // 16 * 16
      rec = min(256, least + 16 * (1 + (k % 2)))
      state = torch.zeros((B, 4), dtype=torch.int32, device='cuda')
      gather = torch.full((2, B, rec), SENTINEL, dtype=torch.uint8, device='cuda')
      flags = torch.zeros((1,), dtype=torch.int32, device='cuda')
      local = torch.zeros((2,), dtype=torch.int32, device='cuda')
      x = _lib.HandoffState()
      x.n_peers, x.rank, x.record_bytes, x.rows, x.first_row = 1, 0, rec, B, 0
      x.d_peer_base[0], x.d_peer_flags[0], x.d_local = (gather.data_ptr(), flags.data_ptr(),
                                                        local.data_ptr())
      for t, f in enumerate(seq):
        dev.show(f)
        reward = rs.randint(-2 ** 31, 2 ** 31 - 1, B).astype(np.int32)
        discount = rs.standard_normal(B).astype(np.float32)
        done, has = rs.randint(0, 2, B).astype(np.uint8), rs.randint(0, 2, B).astype(np.uint8)
        outs = [torch.from_numpy(a).cuda() for a in (reward, has, discount, done)]
        out = _lib.Outputs(dev.boards.data_ptr(), outs[0].data_ptr(), outs[1].data_ptr(),
                           outs[2].data_ptr(), outs[3].data_ptr())
        before = gather[(t + 1) % 2].clone()
        _lib.check(dev.lib.pcl_crop_handoff(
            dev.h, C.byref(spec), dev.boards.data_ptr(), state.data_ptr(), C.byref(out),
            C.byref(x), C.c_void_p(torch.cuda.current_stream().cuda_stream)),
            'pcl_crop_handoff')
        torch.cuda.synchronize()
        got = gather[t % 2].cpu().numpy()
        packed = pack_records(want[t][0], reward, discount, done, has)
        msg = '%s cropper %d t=%d rec %d' % (name, k, t, rec)
        np.testing.assert_array_equal(got[:, :packed.shape[1]], packed, err_msg=msg)
        assert not got[:, packed.shape[1]:].any(), msg + ': padding words not zero'
        assert bool((gather[(t + 1) % 2] == before).all()), msg + ': other part written'
        assert int(local[0]) == t + 1 and int(local[1]) == 0, msg
  finally:
    dev.close()


# ---- attached epilogue -----------------------------------------------------------

@pytest.mark.parametrize('window,margins,pad', [
    ((1, 1), (0, 0), None), ((1, 5), (0, None), ' '), ((3, 5), (1, 2), None),
    ((4, 6), (0, 0), '#'), ((5, 7), (None, None), ' '), ((9, 9), (4, 4), None),
    ((16, 16), (2, 3), None), ((20, 24), (3, 5), ' '), ((255, 257), (2, 3), ' ')], ids=str)
def test_attached_epilogue_matches_the_crop_kernel(window, margins, pad):
  """scrolly_maze's attached cropper (the step kernel's epilogue) writes what crop_kernel
  writes after the same steps, with its own corner state; a drape-tracking spec attached
  afterwards falls back to a crop launch after each step that writes what crop_kernel
  writes, and detaches the epilogue (which would otherwise keep writing into the
  previous cropper's released view and corner state)."""
  import torch
  from pycolab_b200 import batched, levels
  from pycolab_b200.games import scrolly_maze
  arts = [levels.scrolly_maze_level(20 + i, world_shape=(33, 33), board_shape=(16, 16))
          for i in range(2)]
  eng = batched.BatchedEngine([scrolly_maze.make_game(*a) for a in arts], batch=9)
  spec = batched.scrolling_crop_spec(window[0], window[1], 0, pad_char=pad,
                                     scroll_margins=margins)
  drape = batched.scrolling_crop_spec(5, 7, 0, pad_char=' ', scroll_margins=(1, 2),
                                      track=[-1, 1])
  view = eng.attach_cropper(spec)
  assert eng._attached[3]                            # runs inside the step kernel
  state = eng.new_crop_state()
  eng.its_showtime()
  rs = np.random.RandomState(sum(window))
  for t in range(30):
    if t:
      eng.play(torch.from_numpy(rs.randint(0, 5, 9).astype(np.int32)).cuda())
    want = eng.crop(spec, state=state)
    torch.cuda.synchronize()
    assert bool((view == want).all()), t
  # A drape-tracking spec has no epilogue (drape medians need scratch memory): it falls
  # back to a crop launch after each step, and the previous cropper, whose view and
  # state this test now drops, no longer runs inside the step kernel.
  del view
  drape_view = eng.attach_cropper(drape, state=eng.new_crop_state())
  assert not eng._attached[3]
  own = eng.new_crop_state()
  for t in range(20):
    eng.play(torch.from_numpy(rs.randint(0, 5, 9).astype(np.int32)).cuda())
    want = eng.crop(drape, state=own)
    torch.cuda.synchronize()
    assert bool((drape_view == want).all()), t
  eng.attach_cropper(None)


# ---- facade ------------------------------------------------------------------------

ART = ['..............',
       '..%%..........',
       '..%...........',
       '......P.......',
       '..........%%%.',
       '..........%...',
       '..............',
       '..............']


@pytest.mark.parametrize('make', ['scroll_pad', 'scroll', 'fixed_pad', 'fixed_off'])
def test_facade_crops_unoccluded_layers(make):
  """occlusion_in_layers=False: the cropped layers are the observation's un-occluded
  layers cut at the window, pad cells set only in the pad character's layer — not the
  layers of the cropped board."""
  from pycolab_b200 import cropping
  from pycolab_b200.games import fixtures
  walkers = {'P': dict(impassable='', confined=False, egocentric=False)}
  world = ogames.make_fixture_world(ART, '.', walkers, drapes='%')
  game = fixtures.make_game(ART, '.', walkers, drapes='%', occlusion_in_layers=False)
  if make.startswith('scroll'):
    pad = '%' if make == 'scroll_pad' else None
    want_crop = em.ScrollingCrop(5, 7, ['P', '%'], pad_char=pad, scroll_margins=(1, 2))
    got_crop = cropping.ScrollingCropper(5, 7, ['P', '%'], pad_char=pad, scroll_margins=(1, 2))
    want_crop.set_engine(world)
  else:
    corner = (-2, 9) if make == 'fixed_pad' else (20, -30)
    got_crop = cropping.FixedCropper(corner, 5, 7, pad_char='P')
  got_crop.set_engine(game)
  w_out, g_out = world.its_showtime(), game.its_showtime()
  rs = np.random.RandomState(5)
  moves = ['nw'] * 5 + ['se'] * 7 + list(rs.choice(['n', 'e', 's', 'w', 'se', 'nw'], 30))
  occluded = 0
  for t, move in enumerate([None] + moves):
    if move is not None:
      w_out = world.play({'P': em.MOTION_OF_NAME[move]})
      g_out = game.play({'P': move})
    obs = g_out[0]
    got = got_crop.crop(obs)
    if make.startswith('scroll'):
      want_board = want_crop.crop(w_out[0])
      corner = want_crop.corner
    else:
      want_board = em.crop_window(w_out[0], corner, 5, 7, 'P')
    _, want_layers = em.crop_window(obs.board, corner, 5, 7, got_crop._pad_char,
                                    dict(obs.layers))
    np.testing.assert_array_equal(got.board, want_board, err_msg='t=%d' % t)
    assert set(got.layers) == set(want_layers)
    for ch in want_layers:
      np.testing.assert_array_equal(got.layers[ch], want_layers[ch], err_msg='t=%d %s' % (t, ch))
      occluded += int((got.layers[ch] != (got.board == ord(ch))).any())
  if make.startswith('scroll'):
    assert occluded > 0               # some layer differs from the cropped board's


def test_facade_tracking_a_box_world_key_is_not_lowered():
  from pycolab_b200 import cropping
  from pycolab_b200.errors import NotLoweredError
  from pycolab_b200.games import box_world
  game = box_world.make_game(12, (1, 2, 3, 4), (0, 1, 2, 3, 4), (0,), 1,
                             random_state=np.random.RandomState(4))
  game.its_showtime()
  objects = game.batched.object_chars
  assert objects
  crop = cropping.ScrollingCropper(5, 5, [objects[0], box_world.PLAYER], pad_char=None,
                                   scroll_margins=(1, 1))
  crop.set_engine(game)
  with pytest.raises(NotLoweredError, match=repr(objects[0])):
    crop.crop(None)


def test_windows_past_the_cell_limit_are_not_lowered():
  """A 256x256 window (legal upstream) raises NotLoweredError from the facade's crop,
  BatchedEngine.crop, attach_cropper and play_host_async; 255x257 is served."""
  import torch
  from pycolab_b200 import batched, cropping
  from pycolab_b200.errors import NotLoweredError
  from pycolab_b200.games import fixtures
  walkers = {'P': dict(impassable='', confined=False, egocentric=False)}
  game = fixtures.make_game(ART, '.', walkers, drapes='%')
  big = cropping.ScrollingCropper(256, 256, ['P'], pad_char='.', scroll_margins=(0, 0))
  ok = cropping.ScrollingCropper(255, 257, ['P'], pad_char='.', scroll_margins=(0, 0))
  big.set_engine(game)
  ok.set_engine(game)
  obs, _, _ = game.its_showtime()
  with pytest.raises(NotLoweredError):
    big.crop(obs)
  assert ok.crop(obs).board.shape == (255, 257)
  from pycolab_b200 import levels
  from pycolab_b200.games import scrolly_maze
  art = levels.scrolly_maze_level(3, world_shape=(33, 33), board_shape=(16, 16))
  eng = batched.BatchedEngine([scrolly_maze.make_game(*art)], batch=3)
  eng.its_showtime()
  spec = batched.scrolling_crop_spec(256, 256, 0, pad_char=' ', scroll_margins=(0, 0))
  with pytest.raises(NotLoweredError):
    eng.crop(spec)
  with pytest.raises(NotLoweredError):
    eng.attach_cropper(spec)
  assert eng._attached is None
  frames, launches = eng.frames().clone(), eng.launch_count()
  with pytest.raises(NotLoweredError):
    eng.play_host_async(np.zeros(3, np.int32), crop_spec=spec)
  assert bool((eng.frames() == frames).all()) and eng.launch_count() == launches
  eng.play(torch.zeros(3, dtype=torch.int32).cuda())


@pytest.mark.parametrize('track', [[-1], [1, -2], [-2, 1, -1]], ids=str)
def test_play_host_async_refuses_before_stepping(track):
  """A drape-tracking spec given to play_host_async raises before anything is enqueued:
  no env advanced, no launch counted, and the next valid play_host_async / host_wait of
  the same slot works and matches the synchronous path."""
  import torch
  from pycolab_b200 import batched, levels
  from pycolab_b200.errors import NotLoweredError
  from pycolab_b200.games import scrolly_maze
  art = levels.scrolly_maze_level(7, world_shape=(33, 33), board_shape=(16, 16))
  eng = batched.BatchedEngine([scrolly_maze.make_game(*art)], batch=5)
  twin = batched.BatchedEngine([scrolly_maze.make_game(*art)], batch=5)
  eng.its_showtime()
  twin.its_showtime()
  good = batched.scrolling_crop_spec(5, 7, 0, pad_char=' ', scroll_margins=(1, 2))
  bad = batched.scrolling_crop_spec(5, 7, 0, pad_char=' ', scroll_margins=(1, 2), track=track)
  state, twin_state = eng.new_crop_state(), twin.new_crop_state()
  rs = np.random.RandomState(len(track))
  for t in range(6):
    acts = rs.randint(0, 5, 5).astype(np.int32)
    frames, launches = eng.frames().clone(), eng.launch_count()
    with pytest.raises(NotLoweredError):
      eng.play_host_async(acts, slot=t % 2, crop_spec=bad, crop_state=state)
    torch.cuda.synchronize()
    assert bool((eng.frames() == frames).all()) and eng.launch_count() == launches, t
    eng.play_host_async(acts, slot=t % 2, crop_spec=good, crop_state=state)
    view, reward, _, discount, done = eng.host_wait(t % 2)
    twin.play(torch.from_numpy(acts).cuda())
    want = twin.crop(good, state=twin_state).cpu().numpy()
    np.testing.assert_array_equal(view, want, err_msg='t=%d' % t)
    np.testing.assert_array_equal(reward, twin.reward.cpu().numpy())
    np.testing.assert_array_equal(done, twin.done.cpu().numpy())
    assert bool((eng.frames() == frames + 1).all()), t
