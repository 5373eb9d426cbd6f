"""`pcl_crop_observe` and the batched post-processors over cropper windows on the device.

- Direct: a no-program handle over every `crop_cases.CASES` entry (B = 4099, drape
  tracking lists, windows past the board), each cropper called once per frame with its
  own corner state, cycling through element sizes 1 / 2 / 4 / 8, every permute and depths
  1, 32, 33 and 70, board tables and un-occluded layer planes.  The output is written
  between sentinel guards that must come back untouched; it must equal the oracle's
  window (`crop_cases.oracle`) looked up in the table; the corner state must hold the
  oracle's corner after every call; the unknown flag must be set exactly when a byte
  the table does not mark, the pad included, lies in some window.
- The reference goldens (tests/golden/windowobs_*.npz) replayed through
  `observers.crop_observe`, as the engine calls it.
- Engine level: scrolly_maze (4096 envs), better_scrolly_maze's three views, an
  un-occluded fixture game against the facade and the oracle, the unknown pad character,
  and one launch per call.
"""

import ctypes as C
import itertools

import numpy as np
import pytest

import crop_cases as cc
import crop_observe_cases as coc
from oracle import engine_model as em
from test_gpu_crop_grid import _Direct

pytestmark = pytest.mark.gpu

SIZES = (1, 2, 4, 8)
CONTAINER = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}
PERMUTES = [None] + list(itertools.permutations(range(3)))[1:]
DEPTHS = (1, 32, 33, 70)
GUARD = 48
SENTINEL = 0xA5


def _stream():
  import torch
  return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _strides(shape, perm):
  """Element strides of the unpermuted axes of a contiguous [B] + permuted(shape) output."""
  pshape = [shape[i] for i in perm]
  st = [1] * len(pshape)
  for i in range(len(pshape) - 2, -1, -1):
    st[i] = st[i + 1] * pshape[i + 1]
  at = dict((perm[j], st[j]) for j in range(len(perm)))
  return int(np.prod(pshape)), at, pshape


def _combos():
  """(element size, permute or '2d', depth) for every size, permute and depth."""
  out = [(s, p, d) for s in SIZES for p in PERMUTES for d in DEPTHS]
  out += [(s, p, 1) for s in SIZES for p in ('2d', '2d_t')]
  return out


COMBOS = _combos()


def _run_direct(dev, spec, state, curtains, size, permute, depth, table, valid, planes=None,
                plane_of=None, pad_plane=-1):
  """One pcl_crop_observe call into a guarded buffer; returns (output [B] + permuted
  shape, unknown flag)."""
  import torch
  from pycolab_b200 import _lib
  B, r, c = dev.c['B'], spec.rows, spec.cols
  is_3d = permute not in ('2d', '2d_t')
  shape = [depth, r, c] if is_3d else [r, c]
  perm = (list(permute) if permute is not None else [0, 1, 2]) if is_3d else (
      [0, 1] if permute == '2d' else [1, 0])
  per_env, at, pshape = _strides(shape, perm)
  n_bytes = (2 * GUARD + B * per_env) * size
  buf = torch.full((n_bytes,), SENTINEL, dtype=torch.uint8, device='cuda')
  ospec = _lib.ObserveSpec(depth, {1: 0, 2: 5, 4: 1, 8: 3}[size], per_env,
                           at[0] if is_3d else 0, at[1] if is_3d else at[0],
                           at[2] if is_3d else at[1])
  t_table = torch.from_numpy(np.ascontiguousarray(table).view(np.uint8)).cuda()
  t_valid = None if valid is None else torch.from_numpy(valid.astype(np.uint8)).cuda()
  unknown = torch.zeros((1,), dtype=torch.int32, device='cuda')
  pargs = (None, None, -1, 0, 0, 0)
  if planes is not None:
    t_plane_of = torch.tensor(plane_of, dtype=torch.int32, device='cuda')
    pargs = (planes.data_ptr(), t_plane_of.data_ptr(), pad_plane) + tuple(planes.stride()[:3])
  _lib.check(dev.lib.pcl_crop_observe(
      dev.h, C.byref(spec), dev.boards.data_ptr(), None if state is None else state.data_ptr(),
      curtains, C.byref(ospec), t_table.data_ptr(),
      None if t_valid is None else t_valid.data_ptr(), *pargs,
      buf.data_ptr() + GUARD * size, unknown.data_ptr(), _stream()), 'pcl_crop_observe')
  torch.cuda.synchronize()
  raw = buf.cpu().numpy()
  assert (raw[:GUARD * size] == SENTINEL).all(), 'head guard written'
  assert (raw[(GUARD + B * per_env) * size:] == SENTINEL).all(), 'tail guard written'
  got = raw[GUARD * size:(GUARD + B * per_env) * size].view(CONTAINER[size])
  return got.reshape([B] + pshape), int(unknown[0]), perm, is_3d


def _expect(lookup, perm, is_3d):
  """lookup [B, r, c, depth] -> [B] + permuted([depth,] r, c)."""
  if is_3d:
    return np.transpose(np.moveaxis(lookup, 3, 1), [0] + [1 + i for i in perm])
  return np.transpose(lookup[..., 0], [0] + [1 + i for i in perm])


def _curtain_ptrs(dev, spec):
  from pycolab_b200 import _lib
  if not any(code < 0 for code in spec.track):
    return None
  ptrs = (C.c_void_p * _lib.MAX_TRACK)()
  for i, code in enumerate(spec.track):
    if code < 0:
      ptrs[i] = dev.curtains[-code - 1].data_ptr()
  return ptrs


@pytest.mark.parametrize('name', [c['name'] for c in cc.CASES])
def test_direct_grid(name):
  """Every case of the cropper grid through pcl_crop_observe (see the module doc)."""
  import torch
  from pycolab_b200 import _lib
  c = cc.BY_NAME[name]
  seq = cc.frames(c)
  index = [x['name'] for x in cc.CASES].index(name)
  lc = cc.layer_chars(c)
  wants = [cc.oracle(c, k, seq, with_layers=True) for k in c['croppers']]
  specs = [cc.crop_spec(c, k) for k in c['croppers']]
  states = [torch.zeros((c['B'], 4), dtype=torch.int32, device='cuda') if k['state'] == 'own'
            else None for k in c['croppers']]
  rs = np.random.RandomState(index)
  dev = _Direct(c)
  try:
    for t, f in enumerate(seq):
      dev.show(f)
      planes = None
      for k, cropper in enumerate(c['croppers']):
        size, permute, depth = COMBOS[(t * 7 + index * 13 + k * 5) % len(COMBOS)]
        crops, corners, lays = wants[k][t]
        pad = cc.pad_char(c, cropper)
        table = rs.randint(0, 256, (128, depth * size)).astype(np.uint8).view(CONTAINER[size])
        msg = '%s cropper %d t=%d size %d permute %s depth %d' % (name, k, t, size, permute,
                                                                 depth)
        unoccluded = (t + k) % 3 == 2
        if unoccluded:
          if planes is None:
            host = np.zeros((c['B'], len(lc), c['H'], cc.pitch(c['W'])), np.uint8)
            for e in range(c['B']):
              lay = cc.layers(c, f, e)
              for i, ch in enumerate(lc):
                host[e, i, :, :c['W']] = lay[ch]
            planes = torch.from_numpy(host).cuda()
          plane_of = rs.randint(-1, len(lc), depth).tolist()
          pad_plane = lc.find(pad) if pad is not None else -1
          got, unknown, perm, is_3d = _run_direct(
              dev, specs[k], states[k], _curtain_ptrs(dev, specs[k]), size, permute, depth,
              table, None, planes, plane_of, pad_plane)
          bits = np.zeros(crops.shape + (depth,), np.uint8)
          for d, p in enumerate(plane_of):
            if p >= 0:
              bits[..., d] = np.stack([lay[lc[p]] for lay in lays])
          lookup = table[bits, np.arange(depth)]
          assert unknown == 0, msg
        else:
          missing = [None, pad, lc[rs.randint(len(lc))]][rs.randint(3)]
          valid = np.ones(128, bool)
          if missing is not None:
            valid[ord(missing)] = False
          got, unknown, perm, is_3d = _run_direct(
              dev, specs[k], states[k], _curtain_ptrs(dev, specs[k]), size, permute, depth,
              table, valid)
          lookup = table[crops]
          assert unknown == int(not valid[crops].all()), msg + ' unknown flag'
        want = _expect(lookup, perm, is_3d)
        bad = np.nonzero((got != want).reshape(c['B'], -1).any(1))[0]
        assert not len(bad), '%s%s: envs %s differ' % (msg, ' unoccluded' * unoccluded,
                                                       bad[:8].tolist())
        if cropper['kind'] == 'scroll':
          if states[k] is not None:
            np.testing.assert_array_equal(states[k].cpu().numpy()[:, :2], corners,
                                          err_msg=msg + ' corner')
          else:
            slot = dev.plot[:, _lib.P_CROP_R:_lib.P_CROP_C + 1].cpu().numpy()
            np.testing.assert_array_equal(slot, corners, err_msg=msg + ' plot corner')
  finally:
    dev.close()


def test_the_grid_takes_every_combination():
  """Over the grid's calls, every (element size, permute, depth) is taken."""
  seen = set()
  for index, c in enumerate(cc.CASES):
    for t in range(c['T']):
      for k in range(len(c['croppers'])):
        seen.add(COMBOS[(t * 7 + index * 13 + k * 5) % len(COMBOS)])
  assert seen == set(COMBOS)


def test_unknown_flag_counts_the_pad():
  """A FixedCropper window wholly off the board is all pad: the flag is set exactly when
  the table does not mark the pad character."""
  import torch
  c = cc.BY_NAME['b8x14_fixed']
  cropper = c['croppers'][2]                 # at (20, 30): every cell is pad '.'
  assert cropper['corner'] == (20, 30) and cropper['pad'] == 'backdrop'
  spec = cc.crop_spec(c, cropper)
  state = torch.zeros((c['B'], 4), dtype=torch.int32, device='cuda')
  dev = _Direct(c)
  try:
    dev.show(cc.frames(c)[0])
    table = np.arange(128, dtype=np.uint8).reshape(128, 1)
    for marked, want in (('.', 0), ('#', 1), (' .#ABxy', 0), (' #ABxy', 1)):
      valid = np.zeros(128, bool)
      valid[[ord(ch) for ch in marked]] = True
      got, unknown, _, _ = _run_direct(dev, spec, state, None, 1, '2d', 1, table, valid)
      assert unknown == want, marked
      assert (got == ord('.')).all()
  finally:
    dev.close()


# ---- the reference goldens ---------------------------------------------------------

def _tables(proc, present):
  from pycolab_b200 import observers
  if proc['kind'] == 'feature':
    if proc['occluded']:
      return observers.feature_table(proc['layers'], present=present), None, True
    table = np.zeros((128, len(proc['layers'])), np.float32)
    table[1] = 1.0
    return table, None, True
  if proc['kind'] == 'array':
    return observers.value_table(proc['mapping'], np.dtype(proc['dtype']))
  return observers.repaint_table(proc['mapping']), None, False


@pytest.mark.parametrize('name', coc.golden_names())
def test_reference_goldens_replay(name):
  """What the reference's croppers and post-processors returned, through
  observers.crop_observe on the device; each processor keeps its own corner state, as
  each cropper object keeps its own window."""
  import torch
  from pycolab_b200 import observers
  c, seq, want, outs = coc.load_golden(name)
  B, lc = c['B'], cc.layer_chars(c)
  dev = _Direct(c)
  try:
    specs = [cc.crop_spec(c, k) for k in c['croppers']]
    states = dict(((k, p['name']), torch.zeros((B, 4), dtype=torch.int32, device='cuda'))
                  for k in range(len(specs)) for p in coc.PROCESSORS)
    for t, f in enumerate(seq):
      dev.show(f)
      host = np.zeros((B, len(lc), c['H'], cc.pitch(c['W'])), np.uint8)
      for e in range(B):
        lay = cc.layers(c, f, e)
        for i, ch in enumerate(lc):
          host[e, i, :, :c['W']] = lay[ch]
      planes = torch.from_numpy(host).cuda()
      for k, spec in enumerate(specs):
        pad = cc.pad_char(c, c['croppers'][k])
        for proc in coc.PROCESSORS:
          table, valid, is_3d = _tables(proc, lc)
          permute = proc.get('permute')
          unknown = torch.zeros((1,), dtype=torch.int32, device='cuda')
          kw = {}
          if proc['kind'] == 'feature' and not proc['occluded']:
            kw = dict(planes=planes, plane_of=[lc.find(ch) for ch in proc['layers']],
                      pad_plane=lc.find(pad) if pad is not None else -1)
          out = observers.crop_observe(dev.lib, dev.h, spec, dev.boards,
                                       states[(k, proc['name'])], _curtain_ptrs(dev, spec),
                                       table, valid, is_3d, permute, _stream(), unknown, **kw)
          ref_out, ref_raised = outs[(k, proc['name'])]
          got = out.cpu().numpy().view(ref_out.dtype)
          msg = '%s cropper %d %s t=%d' % (name, k, proc['name'], t)
          assert int(unknown[0]) == int(ref_raised[t].any()), msg
          ok = ~ref_raised[t]
          np.testing.assert_array_equal(got[ok], ref_out[t][ok], err_msg=msg)
          if c['croppers'][k]['kind'] == 'scroll':
            np.testing.assert_array_equal(states[(k, proc['name'])].cpu().numpy()[:, :2],
                                          want[k][t][1], err_msg=msg + ' corner')
  finally:
    dev.close()


# ---- engine level ------------------------------------------------------------------

def _batch_oracle(proc, crops):
  out, raised = coc.oracle_apply(proc, crops)
  assert not raised
  return out


def test_scrolly_maze_4096_envs():
  """scrolly_maze at 64 x 64, 4096 envs, 20 steps with quits (auto-resets): each
  post-processor of the 9 x 9 egocentric window equals the oracle's post-processor of
  `crop` from a twin corner state; one launch per call."""
  import torch
  from pycolab_b200 import batched, levels
  from pycolab_b200.games import scrolly_maze
  B = 4096
  eng = batched.BatchedEngine([scrolly_maze.make_game(*levels.scrolly_maze_level(1000 + i))
                               for i in range(4)], batch=B)
  spec = batched.scrolling_crop_spec(9, 9, 0, pad_char=' ', scroll_margins=(None, None))
  states = dict((n, eng.new_crop_state()) for n in ('feat', 'onehot', 'rgb', 'rep', 'twin'))
  chars = eng.chars
  onehot = dict((ch, tuple(int(ch == x) for x in chars)) for ch in chars)
  rgb = dict((ch, float(ord(ch)) / 7) for ch in chars)
  rep = {' ': '.', '#': '%'}
  eng.its_showtime()
  rs = np.random.RandomState(4)
  restarts = 0
  for t in range(21):
    if t:
      a = rs.randint(0, 5, B).astype(np.int32)
      a[rs.random_sample(B) < 0.05] = 5                  # quit: the env restarts
      eng.play(torch.from_numpy(a).cuda())
      restarts += int(eng.done.sum())
    n0 = eng.launch_count()
    feats = eng.to_feature_array(chars, crop_spec=spec, state=states['feat'])
    hot = eng.to_array(onehot, dtype=np.uint8, permute=(1, 2, 0), crop_spec=spec,
                       state=states['onehot'])
    val = eng.to_array(rgb, dtype=np.float32, crop_spec=spec, state=states['rgb'])
    repainted = eng.repaint(rep, crop_spec=spec, state=states['rep'])
    assert eng.launch_count() == n0 + 4, t
    crops = eng.crop(spec, state=states['twin']).cpu().numpy()
    for n in ('feat', 'onehot', 'rgb', 'rep'):
      np.testing.assert_array_equal(states[n].cpu().numpy(), states['twin'].cpu().numpy())
    np.testing.assert_array_equal(
        feats.cpu().numpy(), em.observation_to_feature_array(crops, chars).swapaxes(0, 1),
        err_msg='t=%d' % t)
    want = np.moveaxis(em.observation_to_array(crops, onehot, np.uint8), 0, -1)
    np.testing.assert_array_equal(hot.cpu().numpy(), want, err_msg='t=%d' % t)
    np.testing.assert_array_equal(val.cpu().numpy(),
                                  em.observation_to_array(crops, rgb, np.float32))
    np.testing.assert_array_equal(repainted.cpu().numpy(), em.observation_repaint(crops, rep))
  assert restarts > 0


def test_better_scrolly_three_views():
  """better_scrolly_maze's player, patroller and teaser views, each through to_array and
  to_feature_array with crop_spec, against the post-processors of `crop`."""
  import torch
  import better_scrolly_cases as bsc
  from pycolab_b200 import batched
  art = bsc.open_level(7, (24, 48), 6)
  eng = batched.BatchedEngine([bsc.lowered(art)], batch=37)
  views = [batched.scrolling_crop_spec(10, 30, eng.sprite_chars.index('P'),
                                       initial_offset=(1, -2)),
           batched.scrolling_crop_spec(7, 10, eng.sprite_chars.index('c'), pad_char=' ',
                                       scroll_margins=(None, 3))]
  from pycolab_b200 import _lib
  views.append(_lib.CropSpec(12, 20, -1, ord(' '), 0, 0, 18, 33, 0))
  mapping = dict((ch, (ord(ch), -ord(ch))) for ch in eng.chars)
  states = [[eng.new_crop_state() for _ in range(3)] for _ in views]
  eng.its_showtime()
  rs = np.random.RandomState(1)
  for t in range(25):
    if t:
      eng.play(torch.from_numpy(rs.randint(0, 5, 37).astype(np.int32)).cuda())
    for v, spec in enumerate(views):
      st = states[v]
      feats = eng.to_feature_array(eng.chars + '~', permute=(2, 0, 1), crop_spec=spec,
                                   state=st[0]).cpu().numpy()
      vals = eng.to_array(mapping, dtype=np.int16, crop_spec=spec, state=st[1]).cpu().numpy()
      crops = eng.crop(spec, state=st[2]).cpu().numpy()
      want = em.observation_to_feature_array(crops, eng.chars + '~').swapaxes(0, 1)
      np.testing.assert_array_equal(feats, want.transpose(0, 3, 1, 2), err_msg='%d %d' % (t, v))
      np.testing.assert_array_equal(
          vals, em.observation_to_array(crops, mapping, np.int16).swapaxes(0, 1))


ART = ['..............',
       '..%%..........',
       '..%...........',
       '......P.......',
       '..........%%%.',
       '..........%...',
       '..............',
       '..............']


@pytest.mark.parametrize('pad', ['%', '.', None])
def test_unoccluded_fixture_game(pad):
  """occlusion_in_layers=False: to_feature_array(crop_spec=...) of a batch of the fixture
  game is, for env 0, the facade's ScrollingCropper + ObservationToFeatureArray of the
  single-env Engine, and for every env the oracle's un-occluded layers cut at the
  oracle's corner.  Per call: the tracked drape's curtain export, one pcl_layers and one
  pcl_crop_observe launch."""
  import torch
  from pycolab_b200 import batched, cropping, rendering
  from pycolab_b200.games import fixtures
  from oracle import games as ogames
  walkers = {'P': dict(impassable='', confined=False, egocentric=False)}
  game = fixtures.make_game(ART, '.', walkers, drapes='%', occlusion_in_layers=False)
  B = 6
  eng = batched.BatchedEngine([fixtures.make_game(ART, '.', walkers, drapes='%',
                                                  occlusion_in_layers=False)], batch=B,
                              auto_reset=False)
  worlds = [ogames.make_fixture_world(ART, '.', walkers, drapes='%') for _ in range(B)]
  crops = [em.ScrollingCrop(5, 7, ['P', '%'], pad_char=pad, scroll_margins=(1, 2))
           for _ in range(B)]
  facade = cropping.ScrollingCropper(5, 7, ['P', '%'], pad_char=pad, scroll_margins=(1, 2))
  facade.set_engine(game)
  for w, k in zip(worlds, crops):
    k.set_engine(w)
  spec = batched.scrolling_crop_spec(5, 7, 0, pad_char=pad, scroll_margins=(1, 2),
                                     track=[eng.sprite_chars.index('P') + 1,
                                            -(eng.drape_chars.index('%') + 1)])
  layers = '%P.~%'
  state = eng.new_crop_state()
  obs, _, _ = game.its_showtime()
  eng.its_showtime()
  outs = [w.its_showtime() for w in worlds]
  order = ''.join(eng.game.groups)
  names = ('n', 'ne', 'e', 'se', 's', 'sw', 'w', 'nw', 'stay')
  from pycolab_b200 import _lib
  rs = np.random.RandomState(2)
  moves = [7] * 5 + [3] * 7 + list(rs.randint(0, 9, 30))
  occluded = 0
  for t, m in enumerate([None] + moves):
    if m is not None:
      obs, _, _ = game.play(names[m])
      rows = np.zeros((B, len(order) + 2 * _lib.FIXTURE_DIRECTIVES), np.int32)
      per_env = [(m + e) % 9 if t > 12 else m for e in range(B)]
      rows[:, :len(order)] = np.array(per_env)[:, None]
      eng.play(torch.from_numpy(rows).cuda())
      outs = [w.play({'P': em.MOTION_OF_NAME[names[a]]}) for w, a in zip(worlds, per_env)]
    n0 = eng.launch_count()
    got = eng.to_feature_array(layers, crop_spec=spec, state=state).cpu().numpy()
    assert eng.launch_count() == n0 + 3, t   # the tracked drape's curtain, the layers, the window
    np.testing.assert_array_equal(
        got[0], rendering.ObservationToFeatureArray(layers)(facade.crop(obs)),
        err_msg='facade t=%d' % t)
    for e in range(B):
      board = outs[e][0]
      lay = em.unoccluded_layers_of(worlds[e].backdrop, worlds[e].things, 'P.%')
      cut_board = crops[e].crop(board)
      _, cut = em.crop_window(board, crops[e].corner, 5, 7, pad, lay)
      want = em.observation_to_feature_array(cut_board, layers, observation_layers=cut)
      np.testing.assert_array_equal(got[e], want, err_msg='env %d t=%d' % (e, t))
      occluded += int(any((want[i] != (cut_board == ord(layers[i]))).any() for i in range(3)))
  assert occluded > 0


def test_to_array_raises_on_an_unmapped_pad():
  """A window past the board shows the pad character: to_array raises when the mapping
  lacks it, even though no board cell holds it; repaint and to_feature_array do not."""
  import torch
  from pycolab_b200 import _lib, batched
  from pycolab_b200.games.classics import four_rooms
  eng = batched.BatchedEngine([four_rooms.make_game()], batch=5)
  eng.its_showtime()
  board_chars = set(eng.chars)
  fixed = _lib.CropSpec(5, 7, -1, ord('~'), 0, 0, -3, -4, 0)     # '~': pad cells only
  mapping = dict((ch, ord(ch)) for ch in board_chars)
  with pytest.raises(RuntimeError):
    eng.to_array(mapping, dtype=np.int32, crop_spec=fixed)
  got = eng.to_array(dict(mapping, **{'~': -1}), dtype=np.int32, crop_spec=fixed).cpu().numpy()
  assert (got[:, :3, :] == -1).all() and (got[:, :, :4] == -1).all()
  assert (got[:, 3:, 4:] >= 0).all()
  eng.repaint({'~': '#'}, crop_spec=fixed)
  eng.to_feature_array('~#', crop_spec=fixed)
  inner = _lib.CropSpec(3, 3, -1, ord('~'), 0, 0, 1, 1, 0)
  eng.to_array(mapping, dtype=np.int32, crop_spec=inner)        # all on the board: no raise
  torch.cuda.synchronize()
