"""Host side of the observation post-processors, no GPU: the tables
`observers` builds for pcl_observe, and the oracle's post-processors against
upstream `pycolab.rendering` over the dtypes, depths and bytes the device grid
(test_gpu_observers_grid.py) uses."""

import warnings

import numpy as np
import pytest

import refdriver
from oracle import engine_model as em
from pycolab_b200 import observers

import test_gpu_observers_grid as grid


@pytest.mark.parametrize('kind', grid.DTYPES + grid.INFERRED)
def test_value_table_dtype_and_size(kind):
  rs = np.random.RandomState(1)
  for depth in (0, 3, 33):
    if (kind == 'tuple' and depth == 0) or (kind in ('int', 'float') and depth):
      continue
    mapping, dt = grid._mapping(kind, depth, rs, missing='xyz')
    with warnings.catch_warnings():
      warnings.simplefilter('ignore')
      table, valid, is_3d = observers.value_table(mapping, dt)
    want_dt = dt if dt is not None else np.array(next(iter(mapping.values()))).dtype
    assert table.dtype == want_dt and table.shape == (128, max(depth, 1))
    assert is_3d == (depth > 0)
    assert valid.dtype == np.uint8 and valid.sum() == 125
    assert not valid[[ord('x'), ord('y'), ord('z')]].any()
    assert not table[ord('x')].view(grid._unsigned(table.dtype)).any()
    # each row holds exactly what upstream's masked assignment stores
    board = np.array([[ord('A'), ord('~')]], np.uint8)
    with warnings.catch_warnings():
      warnings.simplefilter('ignore')
      want = em.observation_to_array(board, mapping, dt)
    want = want.reshape(max(depth, 1), 2).T
    np.testing.assert_array_equal(table[[ord('A'), ord('~')]].view(grid._unsigned(table.dtype)),
                                  want.view(grid._unsigned(want.dtype)))


@pytest.mark.parametrize('dtype', [np.complex128, np.complex64, object, 'U1', 'S1',
                                   'datetime64[s]', np.longdouble])
def test_value_table_refuses_other_types(dtype):
  with pytest.raises(TypeError):
    observers.value_table({'a': 1, 'b': 2}, dtype)
  with pytest.raises(TypeError):
    observers.value_table({'a': 1j, 'b': 2j})                  # inferred complex128


def test_plane_chunks():
  for depth in (1, 31, 32, 33, 64, 65, 95):
    chunks = observers.plane_chunks(depth)
    assert all(1 <= n <= observers.MAX_PLANES for _, n in chunks)
    assert [k for k, _ in chunks] == list(range(0, depth, 32))
    assert sum(n for _, n in chunks) == depth


def test_feature_and_repaint_tables():
  t = observers.feature_table('ab\xc8c', present=set('abx'))
  assert t.dtype == np.float32 and t.shape == (128, 4)
  assert t[ord('a'), 0] == 1 and t[ord('b'), 1] == 1 and t.sum() == 2   # '\xc8', 'c': zeros
  t = observers.repaint_table({'a': 'b', '#': ' '})
  assert t.dtype == np.uint8 and t.shape == (128, 1)
  assert t[ord('a'), 0] == ord('b') and t[ord('#'), 0] == ord(' ') and t[ord('q'), 0] == ord('q')


needs_ref = pytest.mark.skipif(not refdriver.available(), reason='reference not present')


def _ref():
  refdriver._import()
  from pycolab import rendering
  return rendering


@needs_ref
@pytest.mark.parametrize('kind', grid.DTYPES + grid.INFERRED)
def test_oracle_to_array_matches_upstream(kind):
  ref = _ref()
  rs = np.random.RandomState(2)
  for (H, W), depth, permute in [((7, 17), 0, None), ((1, 1), 0, (1, 0)), ((3, 4), 3, (1, 2, 0)),
                                 ((7, 15), 33, (2, 0, 1)), ((7, 16), 64, None)]:
    if (kind == 'tuple') == (depth == 0) or (kind in ('int', 'float') and depth):
      continue
    board = grid._boards(rs, 1, H, W, high=False)[0, :, :W]
    mapping, dt = grid._mapping(kind, depth, rs)
    obs = ref.Observation(board=board, layers={})
    with warnings.catch_warnings():
      warnings.simplefilter('ignore')
      want = ref.ObservationToArray(mapping, dtype=dt, permute=permute)(obs)
      got = em.observation_to_array(board, mapping, dt, permute)
    assert got.dtype == want.dtype and got.shape == want.shape
    np.testing.assert_array_equal(got.view(grid._unsigned(got.dtype)),
                                  want.view(grid._unsigned(want.dtype)))
    high = board.copy()
    high[-1, -1] = 200
    for f in (lambda: ref.ObservationToArray(mapping, dtype=dt)(ref.Observation(high, {})),
              lambda: em.observation_to_array(high, mapping, dt)):
      with pytest.raises(RuntimeError), warnings.catch_warnings():
        warnings.simplefilter('ignore')
        f()


@needs_ref
def test_oracle_repaint_and_features_match_upstream():
  ref = _ref()
  rs = np.random.RandomState(3)
  printable = ''.join(chr(c) for c in range(32, 127))
  mapping = {'a': 'b', '#': ' ', chr(0): chr(127)}
  for (H, W) in grid.BOARDS:
    board = grid._boards(rs, 1, H, W, high=False)[0, :, :W]
    chars = set(printable[::2])
    layers = {c: board == ord(c) for c in chars}
    obs = ref.Observation(board=board, layers=layers)
    np.testing.assert_array_equal(ref.ObservationCharacterRepainter(mapping)(obs).board,
                                  em.observation_repaint(board, mapping))
    for feats, permute in [(printable[:36], None), (printable, (1, 2, 0))]:
      np.testing.assert_array_equal(
          ref.ObservationToFeatureArray(feats, permute=permute)(obs),
          em.observation_to_feature_array(board, feats, permute, observation_layers=layers))
    high = grid._boards(rs, 1, H, W)[0, :, :W]          # bytes >= 128 too
    high[0, 0] = 200
    obs = ref.Observation(board=high, layers={c: high == ord(c) for c in chars})
    with pytest.raises(RuntimeError):
      ref.ObservationCharacterRepainter(mapping)(obs)
    with pytest.raises(RuntimeError):
      em.observation_repaint(high, mapping)
    np.testing.assert_array_equal(
        ref.ObservationToFeatureArray(printable)(obs),
        em.observation_to_feature_array(high, printable, observation_layers=obs.layers))
    np.testing.assert_array_equal(                      # occluded default: board == c
        ref.ObservationToFeatureArray(printable)(obs),
        em.observation_to_feature_array(high, printable) * np.array(
            [c in chars for c in printable], np.float32)[:, None, None])
