"""Observation post-processors on the device vs the oracle, bit for bit.

`observe_kernel` (csrc/observe.cu) behind `pcl_observe`, reached three ways: the C
entry point on a no-program handle, the facade classes (`rendering.ObservationTo*`,
`ObservationCharacterRepainter`) and `BatchedEngine.to_array / to_feature_array /
repaint`.  The grid covers every element size and kind NumPy offers for values,
depths on both sides of one launch's 32 planes, every `permute`, boards whose
width is not a multiple of 4 or of the 16-byte pitch, every byte value 0..255 on
the board, and a batch large enough for the kernel's grid-stride loop to take a
second pass.  Outputs are compared as bit patterns, so -0.0, NaN payloads and
float16 / float64 rounding all count.
"""

import ctypes as C
import itertools
import warnings

import numpy as np
import pytest

import golden_cases as gc
from oracle import engine_model as em

pytestmark = pytest.mark.gpu

DTYPES = ['bool', 'int8', 'uint8', 'int16', 'uint16', 'float16', 'int32', 'uint32',
          'float32', 'int64', 'uint64', 'float64']
INFERRED = ['int', 'float', 'tuple']           # dtype=None: inferred from the first value
SPECIAL = [0.1, 1e300, 5e-324, float('inf'), -float('inf'), float('nan'), -0.0, 2 ** 40,
           -2 ** 63, 2 ** 64 - 1, -128, 65504, 2]
BOARDS = [(1, 1), (1, 17), (3, 4), (7, 15), (7, 16), (7, 17), (64, 64), (65, 129), (128, 128)]
PERMS3 = list(itertools.permutations(range(3)))
SENTINEL = 0xA5
GUARD = 64                    # elements of sentinel on each side of the output view


def _pitch(W):
  return (W + 15) // 16 * 16


def _unsigned(dt):
  return np.dtype('u%d' % np.dtype(dt).itemsize)


def _accepted(dt):
  """The special values NumPy stores into `dt` (upstream's masked assignment);
  the others raise there as they do upstream."""
  out = []
  for v in SPECIAL:
    a = np.zeros(2, dt)
    try:
      with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        a[np.array([True, False])] = v
    except (OverflowError, ValueError, TypeError):
      continue
    out.append(v)
  return out


def _mapping(kind, depth, rs, missing=''):
  """A value mapping of every ASCII character but `missing` for dtype `kind`
  (None-inferred kinds give Python values); returns (mapping, dtype argument)."""
  if kind in INFERRED:
    dt = None
    if kind == 'int':
      vals = [int(v) for v in rs.randint(-2 ** 62, 2 ** 62, size=128, dtype=np.int64)]
      vals[:3] = [-2 ** 63, 2 ** 63 - 1, 0]
      mapping = {chr(i): vals[i] for i in range(128)}
    elif kind == 'float':
      vals = [float(v) for v in rs.standard_normal(128) * 1e10]
      vals[:len(SPECIAL)] = [float(v) for v in SPECIAL]
      mapping = {chr(i): vals[i] for i in range(128)}
    else:
      mapping = {chr(i): tuple(int(v) for v in rs.randint(-2 ** 40, 2 ** 40, size=depth))
                 for i in range(128)}
  else:
    dt = np.dtype(kind)
    specials = _accepted(dt)
    u = _unsigned(dt)
    bits = rs.randint(0, 256, size=(128, max(depth, 1) * dt.itemsize)).astype(np.uint8)
    rand = bits.view(u).view(dt) if dt != np.bool_ else (bits[:, ::1] & 1).astype(bool)
    rand = rand.reshape(128, -1)[:, :max(depth, 1)]

    def val(i, d):
      k = i * 7 + d
      if k % 3 == 0 and specials:
        return specials[(k // 3) % len(specials)]
      v = rand[i, d]
      return v.item() if dt.kind != 'f' else float(v) if np.isfinite(v) else 1.5
    if depth == 0:
      mapping = {chr(i): val(i, 0) for i in range(128)}
    else:
      mapping = {chr(i): tuple(val(i, d) for d in range(depth)) for i in range(128)}
  for ch in missing:
    del mapping[ch]
  return mapping, dt


def _boards(rs, B, H, W, allowed=None, high=True):
  """u8 [B, H, pitch]: in-board cells drawn from `allowed` (default every byte
  0..255, each placed at least once when the batch has room); pad columns hold
  bytes >= 128, outside every mapping."""
  pitch = _pitch(W)
  boards = rs.randint(128, 256, size=(B, H, pitch)).astype(np.uint8)
  pool = np.arange(256 if high else 128) if allowed is None else np.asarray(allowed)
  cells = rs.choice(pool, size=(B, H, W)).astype(np.uint8)
  flat = cells.reshape(-1)
  if allowed is None and flat.size >= len(pool):
    flat[rs.permutation(flat.size)[:len(pool)]] = pool
  boards[:, :, :W] = cells
  return boards


def _handle(B, H, W):
  from pycolab_b200 import _lib
  spec = _lib.Spec()
  spec.abi_version, spec.program = _lib.ABI_VERSION, _lib.PROG_NONE
  spec.rows, spec.cols, spec.pitch = H, W, _pitch(W)
  h = C.c_void_p()
  _lib.check(_lib.load().pcl_create(C.byref(spec), B, 0, C.byref(h)), 'pcl_create')
  return h


def _direct(boards, W, table, valid, is_3d, permute):
  """pcl_observe on a no-program handle; the output is a view in the middle of a
  sentinel-filled allocation.  Returns (output as table.dtype, unknown flag)."""
  import torch
  from pycolab_b200 import _lib
  lib = _lib.load()
  B, H, _ = boards.shape
  depth, size = table.shape[1], table.dtype.itemsize
  base = [depth, H, W] if is_3d else [H, W]
  perm = list(permute) if permute is not None else list(range(len(base)))
  shape = [B] + [base[i] for i in perm]
  n = int(np.prod(shape))
  buf = torch.full(((2 * GUARD + n) * size,), SENTINEL, dtype=torch.uint8, device='cuda')
  out = buf.view(getattr(torch, _unsigned(table.dtype).name))[GUARD:GUARD + n].view(shape)
  st = out.stride()
  at = {d: st[1 + perm.index(d)] for d in range(len(base))}
  code = {1: 0, 2: 5, 4: 1, 8: 3}[size]
  spec = _lib.ObserveSpec(depth, code, st[0], at[0] if is_3d else 0,
                          at[1] if is_3d else at[0], at[2] if is_3d else at[1])
  t_table = torch.from_numpy(np.ascontiguousarray(table).view(_unsigned(table.dtype))).cuda()
  t_valid = torch.from_numpy(valid).cuda()
  t_board = torch.from_numpy(boards).cuda()
  unknown = torch.zeros((1,), dtype=torch.int32, device='cuda')
  h = _handle(B, H, W)
  try:
    _lib.check(lib.pcl_observe(h, C.byref(spec), t_table.data_ptr(), t_valid.data_ptr(),
                               t_board.data_ptr(), out.data_ptr(), unknown.data_ptr(),
                               C.c_void_p(torch.cuda.current_stream().cuda_stream)),
               'pcl_observe')
    torch.cuda.synchronize()
  finally:
    lib.pcl_destroy(h)
  raw = buf.cpu().numpy()
  guard = GUARD * size
  assert (raw[:guard] == SENTINEL).all() and (raw[-guard:] == SENTINEL).all(), 'guard written'
  return out.cpu().numpy().view(table.dtype), bool(int(unknown[0]))


def _expected(boards, W, mapping, dtype, is_3d, permute):
  """The oracle over every board, cells outside the mapping as zero elements
  (upstream raises on them; the kernel writes zeros and flags them)."""
  B, H, _ = boards.shape
  stacked = boards[:, :, :W].reshape(B * H, W).copy()
  outside = np.isin(stacked, [ord(c) for c in mapping], invert=True)
  stacked[outside] = ord(next(iter(mapping)))
  with warnings.catch_warnings():
    warnings.simplefilter('ignore')
    want = em.observation_to_array(stacked, mapping, dtype)
  want = want.view(_unsigned(want.dtype)).copy()
  if is_3d:
    want[:, outside] = 0
    want = want.reshape(-1, B, H, W).transpose(1, 0, 2, 3)
  else:
    want[outside] = 0
    want = want.reshape(B, H, W)
  if permute is not None:
    want = want.transpose([0] + [1 + p for p in permute])
  return want, bool(outside.any())


def _check_direct(boards, W, mapping, dtype, permute):
  from pycolab_b200 import observers
  with warnings.catch_warnings():
    warnings.simplefilter('ignore')
    table, valid, is_3d = observers.value_table(mapping, dtype)
  got, unknown = _direct(boards, W, table, valid, is_3d, permute)
  want, outside = _expected(boards, W, mapping, dtype, is_3d, permute)
  assert got.shape == want.shape
  np.testing.assert_array_equal(got.view(_unsigned(got.dtype)), want)
  assert unknown == outside


@pytest.mark.parametrize('kind', DTYPES + INFERRED)
def test_direct_every_dtype(kind):
  """Each value type through pcl_observe: scalars and 3-vectors, small, ragged and
  wide boards, every byte on the board."""
  rs = np.random.RandomState(len(kind) * 31 + 7)
  for (H, W), B in [((1, 1), 1), ((7, 17), 5), ((65, 129), 1)]:
    boards = _boards(rs, B, H, W)
    for depth in (0, 3):
      if kind == 'tuple' and depth == 0:
        continue
      if kind in ('int', 'float') and depth == 3:
        continue
      mapping, dt = _mapping(kind, depth, rs)
      permute = (None, (1, 0))[B % 2] if depth == 0 else PERMS3[(H + W) % 6]
      _check_direct(boards, W, mapping, dt, permute)


@pytest.mark.parametrize('depth', [1, 3, 4, 31, 32])
@pytest.mark.parametrize('permute', PERMS3)
def test_direct_depths_and_orders(depth, permute):
  kind = ['uint8', 'float16', 'float32', 'float64', 'int16'][PERMS3.index(permute) % 5]
  rs = np.random.RandomState(depth * 10 + PERMS3.index(permute))
  for (H, W), B in [((7, 15), 5), ((3, 4), 1)]:
    mapping, dt = _mapping(kind, depth, rs)
    _check_direct(_boards(rs, B, H, W), W, mapping, dt, permute)


@pytest.mark.parametrize('shape', BOARDS, ids=['%dx%d' % s for s in BOARDS])
@pytest.mark.parametrize('B', [1, 5])
def test_direct_board_shapes(shape, B):
  H, W = shape
  rs = np.random.RandomState(H * 1000 + W + B)
  boards = _boards(rs, B, H, W)
  for kind, depth, permute in [('float64', 2, (1, 2, 0)), ('uint16', 3, (2, 0, 1)),
                               ('uint8', 0, (1, 0)), ('float32', 5, None)]:
    mapping, dt = _mapping(kind, depth, rs)
    _check_direct(boards, W, mapping, dt, permute)


def test_direct_second_pass_of_the_grid_stride_loop():
  """B * H * pitch / 4 words beyond one wave of 2112 blocks of 256 threads: the one
  character outside the mapping sits in the last env, which only the second pass
  of the loop reads."""
  H, W, B = 64, 60, 600
  assert B * H * _pitch(W) // 4 > 2112 * 256
  assert (B - 1) * H * _pitch(W) // 4 >= 2112 * 256
  rs = np.random.RandomState(5)
  mapping, dt = _mapping('int16', 2, rs, missing='~')
  allowed = [ord(c) for c in mapping]
  boards = _boards(rs, B, H, W, allowed=allowed)
  _check_direct(boards, W, mapping, dt, (2, 0, 1))          # nothing unknown
  boards[B - 1, H - 1, W - 2] = ord('~')
  _check_direct(boards, W, mapping, dt, None)               # ... and now the last env


def test_direct_unknown_flag_is_exact():
  """d_unknown: not set by bytes >= 128 in the pad columns, set by one in-board byte
  >= 128 or one character outside the mapping; such cells come out as zeros."""
  rs = np.random.RandomState(11)
  mapping, dt = _mapping('float32', 3, rs, missing='Q')
  allowed = [ord(c) for c in mapping]
  for (H, W) in [(7, 17), (1, 1), (3, 4)]:
    boards = _boards(rs, 3, H, W, allowed=allowed)
    _check_direct(boards, W, mapping, dt, None)
    for bad in (ord('Q'), 128, 200, 255):
      b = boards.copy()
      b[2, H - 1, W - 1] = bad
      _check_direct(b, W, mapping, dt, (1, 2, 0))


# ---- the facade classes --------------------------------------------------------

def _facade_obs(board, chars=None):
  from pycolab_b200 import rendering
  chars = set(chr(c) for c in np.unique(board) if c < 128) if chars is None else chars
  return rendering.Observation(board=board, layers=rendering.LazyLayers(board, chars))


def _bits(a):
  return np.asarray(a).view(_unsigned(np.asarray(a).dtype))


@pytest.mark.parametrize('kind', DTYPES + INFERRED)
def test_facade_to_array_every_dtype(kind):
  from pycolab_b200 import rendering
  rs = np.random.RandomState(3 + len(kind))
  board = _boards(rs, 1, 7, 17, high=False)[0, :, :17]
  for depth, permute in [(0, None), (0, (1, 0)), (3, (1, 2, 0)), (33, (2, 1, 0))]:
    if (kind == 'tuple') == (depth == 0) or (kind in ('int', 'float') and depth):
      continue
    mapping, dt = _mapping(kind, depth, rs)
    with warnings.catch_warnings():
      warnings.simplefilter('ignore')
      got = rendering.ObservationToArray(mapping, dtype=dt, permute=permute)(_facade_obs(board))
      want = em.observation_to_array(board, mapping, dt, permute)
    assert got.dtype == want.dtype and got.shape == want.shape
    np.testing.assert_array_equal(_bits(got), _bits(want))


@pytest.mark.parametrize('depth', [33, 64])
@pytest.mark.parametrize('permute', PERMS3)
def test_facade_to_array_beyond_one_launch(depth, permute):
  """More than 32 planes: one launch per 32 planes, each at its own plane offset."""
  from pycolab_b200 import rendering
  kind = ['float64', 'uint8', 'float16', 'int32', 'uint64', 'bool'][PERMS3.index(permute)]
  rs = np.random.RandomState(depth + PERMS3.index(permute))
  for H, W in [(7, 15), (65, 129)]:
    board = _boards(rs, 1, H, W, high=False)[0, :, :W]
    mapping, dt = _mapping(kind, depth, rs)
    with warnings.catch_warnings():
      warnings.simplefilter('ignore')
      got = rendering.ObservationToArray(mapping, dtype=dt, permute=permute)(_facade_obs(board))
      want = em.observation_to_array(board, mapping, dt, permute)
    assert got.shape == want.shape
    np.testing.assert_array_equal(_bits(got), _bits(want))


PRINTABLE = ''.join(chr(c) for c in range(32, 127))


@pytest.mark.parametrize('layers', [PRINTABLE[:36], PRINTABLE], ids=['36', '95'])
@pytest.mark.parametrize('permute', [None] + PERMS3)
def test_facade_feature_arrays(layers, permute):
  """One-hot planes over 36 and over all 95 printable characters; bytes >= 128 on
  the board (a canvas painted with paint_all_of may hold them) are in no plane."""
  from pycolab_b200 import rendering
  rs = np.random.RandomState(len(layers))
  for H, W in [(1, 1), (7, 17), (65, 129)]:
    board = _boards(rs, 1, H, W)[0, :, :W]
    chars = set(PRINTABLE[::2])                     # the observation's layers
    obs = _facade_obs(board, chars)
    got = rendering.ObservationToFeatureArray(layers, permute=permute)(obs)
    want = em.observation_to_feature_array(board, layers, permute,
                                           observation_layers={c: board == ord(c) for c in chars})
    assert got.dtype == np.float32 and got.shape == want.shape
    np.testing.assert_array_equal(_bits(got), _bits(want))


def test_facade_feature_array_copies_other_layers():
  """Layers that are not `board == c` (here: made up) are copied, as upstream."""
  from pycolab_b200 import rendering
  rs = np.random.RandomState(2)
  board = _boards(rs, 1, 7, 17, high=False)[0, :, :17]
  layers = {c: rs.random_sample((7, 17)) < 0.5 for c in 'ab#'}
  obs = rendering.Observation(board=board, layers=layers)
  got = rendering.ObservationToFeatureArray('#xab', permute=(1, 2, 0))(obs)
  want = em.observation_to_feature_array(board, '#xab', (1, 2, 0), observation_layers=layers)
  np.testing.assert_array_equal(got, want)


def test_facade_repainter_high_bytes_raise():
  from pycolab_b200 import rendering
  rs = np.random.RandomState(4)
  mapping = {'a': 'b', '#': ' ', chr(0): chr(127)}
  board = _boards(rs, 1, 7, 17, high=False)[0, :, :17]
  rep = rendering.ObservationCharacterRepainter(mapping)(_facade_obs(board))
  np.testing.assert_array_equal(rep.board, em.observation_repaint(board, mapping))
  for bad in (128, 200, 255):
    b = board.copy()
    b[6, 16] = bad
    with pytest.raises(RuntimeError):
      em.observation_repaint(b, mapping)
    with pytest.raises(RuntimeError):
      rendering.ObservationCharacterRepainter(mapping)(_facade_obs(b))


# ---- BatchedEngine -------------------------------------------------------------

def _engine_with_boards(boards, W):
  """A one-walker fixture game of the boards' shape, its device boards replaced."""
  import torch
  from pycolab_b200 import batched
  from pycolab_b200.games import fixtures
  B, H, _ = boards.shape
  art = ['P' + ' ' * (W - 1)] + [' ' * W] * (H - 1)
  eng = batched.BatchedEngine([fixtures.make_game(art, ' ', {'P': {}})], batch=B,
                              auto_reset=False)
  eng.its_showtime()
  eng._board.copy_(torch.from_numpy(boards))
  return eng


@pytest.mark.parametrize('shape', [(3, 4), (7, 17), (65, 129)], ids=str)
def test_batched_post_processors(shape):
  H, W = shape
  B = 5
  rs = np.random.RandomState(H + W)
  boards = _boards(rs, B, H, W, high=False)
  eng = _engine_with_boards(boards, W)
  for i, (kind, depth, permute) in enumerate([('float16', 0, (1, 0)), ('bool', 3, (1, 2, 0)),
                                              ('int', 0, None), ('uint64', 40, (2, 0, 1)),
                                              ('int8', 64, None), ('tuple', 2, (0, 2, 1))]):
    mapping, dt = _mapping(kind, depth, rs)
    with warnings.catch_warnings():
      warnings.simplefilter('ignore')
      got = eng.to_array(mapping, dtype=dt, permute=permute).cpu().numpy()
      for e in range(B):
        want = em.observation_to_array(boards[e, :, :W], mapping, dt, permute)
        assert got[e].dtype == want.dtype and got[e].shape == want.shape
        np.testing.assert_array_equal(_bits(got[e]), _bits(want), err_msg='%d env %d' % (i, e))
  feats = eng.to_feature_array(PRINTABLE, permute=(1, 2, 0)).cpu().numpy()
  rep = eng.repaint({'a': 'b', ' ': '#'}).cpu().numpy()
  for e in range(B):
    board = boards[e, :, :W]
    game_layers = {c: board == ord(c) for c in eng.chars}
    np.testing.assert_array_equal(feats[e], em.observation_to_feature_array(
        board, PRINTABLE, (1, 2, 0), observation_layers=game_layers))
    np.testing.assert_array_equal(rep[e], em.observation_repaint(board, {'a': 'b', ' ': '#'}))
  boards[B - 1, H - 1, W - 1] = 130
  eng._board.copy_(__import__('torch').from_numpy(boards))
  with pytest.raises(RuntimeError):
    eng.to_array(_mapping('uint8', 0, rs)[0])


# ---- the reference's own answers -----------------------------------------------

def _kat_calls():
  import json
  import os
  path = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden',
                      'reference_engine_kats.json')
  with open(path) as f:
    return json.load(f)['observers']


@pytest.mark.parametrize('i', range(14))
def test_reference_observer_calls_on_the_device(i):
  """The 14 post-processor calls of the reference's engine_test.py, replayed
  through the facade classes; their outputs are the reference's."""
  import reference_kats as rk
  from pycolab_b200 import rendering
  call = _kat_calls()[i]
  board = rk.u8(call['board'])
  want = np.array(call['out'], dtype=call['out_dtype']).reshape(call['out_shape'])
  args, kwargs = call['args'], call['kwargs']
  permute = kwargs.get('permute')
  permute = None if permute is None else tuple(permute)
  obs = _facade_obs(board, set(chr(c) for c in np.unique(board)))
  if call['kind'] == 'ObservationCharacterRepainter':
    got = rendering.ObservationCharacterRepainter(args[0])(obs).board
  elif call['kind'] == 'ObservationToArray':
    mapping = {k: (tuple(v) if isinstance(v, list) else v) for k, v in args[0].items()}
    dt = np.dtype(kwargs['dtype']) if kwargs.get('dtype') else None
    got = rendering.ObservationToArray(mapping, dtype=dt, permute=permute)(obs)
  else:
    got = rendering.ObservationToFeatureArray(args[0], permute=permute)(obs)
  assert got.shape == want.shape and got.dtype == want.dtype, (got.dtype, want.dtype)
  np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize('name', gc.names('fixture_unoccluded_'))
def test_unoccluded_feature_arrays_golden(name):
  """occlusion_in_layers=False: the feature array is the golden's un-occluded
  layers, through the facade Engine and through a BatchedEngine of the game."""
  import torch
  from pycolab_b200 import _lib, batched, rendering
  from pycolab_b200.games import fixtures
  g = gc.load(name)
  kw, cfg = gc.fixture_kwargs(g)
  args = (kw['art'], kw['what_lies_beneath'], kw['walkers'], kw['scrollys'], kw['drapes'],
          kw['update_schedule'], kw['z_order'])
  game = fixtures.make_game(*args, occlusion_in_layers=False)
  eng = batched.BatchedEngine([fixtures.make_game(*args, occlusion_in_layers=False)],
                              batch=2, auto_reset=False)
  chars = cfg['layer_chars']
  layers = chars + '~'                       # '~' is no character of the game: zeros
  names = ('n', 'ne', 'e', 'se', 's', 'sw', 'w', 'nw', 'stay')
  order = ''.join(eng.game.groups)
  obs, _, _ = game.its_showtime()
  eng.its_showtime()
  for t in range(len(g['actions']) + 1):
    want = np.concatenate([g['layers'][t].astype(np.float32),
                           np.zeros((1,) + obs.board.shape, np.float32)])
    got = rendering.ObservationToFeatureArray(layers)(obs)
    np.testing.assert_array_equal(got, want, err_msg='facade t=%d' % t)
    feats = eng.to_feature_array(layers, permute=(1, 2, 0)).cpu().numpy()
    for e in range(2):
      np.testing.assert_array_equal(feats[e], want.transpose(1, 2, 0),
                                    err_msg='batched env %d t=%d' % (e, t))
    if t < len(g['actions']):
      a = int(g['actions'][t])
      obs, _, _ = game.play(names[a])
      rows = np.zeros((2, len(order) + 2 * _lib.FIXTURE_DIRECTIVES), np.int32)
      rows[:, :len(order)] = a                 # everybody: the same motion, no directives
      eng.play(torch.from_numpy(rows).cuda())
