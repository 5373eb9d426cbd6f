"""Episode returns (`pcl_bind_episodes`, `pcl_rollout_episodes`, `track_episodes=`) without
a GPU.

- The ctypes mirror of `pcl_episode_rec` and the new entry points against include/pcl.h.
- C-boundary refusals on handles that reach no device (device -1, made-up addresses),
  before anything is enqueued.
- The facade's argument checks, which run before anything needs CUDA.
- The host reference (tests/episode_reference.py) on crafted sequences.
"""

import ctypes as C
import os
import re

import numpy as np
import pytest

import boundary_sweep
import episode_reference as ref
from pycolab_b200 import _lib

FAKE = boundary_sweep.FAKE
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header():
  with open(os.path.join(ROOT, 'include', 'pcl.h')) as f:
    return f.read()


def test_ctypes_mirror_matches_the_header():
  header = _header()
  body = re.search(r'typedef struct pcl_episode_rec \{(.*?)\} pcl_episode_rec;', header, re.S)
  names = re.findall(r'(\w+);', body.group(1))
  assert names == [name for name, _ in _lib.EpisodeRec._fields_] == ['d_return', 'd_length']
  lib = _lib.load()
  assert lib.pcl_episode_rec_size() == C.sizeof(_lib.EpisodeRec) == 2 * 8
  assert lib.pcl_rollout_rec_size() == C.sizeof(_lib.RolloutRec) == 17 * 8   # unchanged
  assert re.search(r'int pcl_bind_episodes\(pcl_handle\* h, double\* d_return\);', header)
  assert re.search(r'int pcl_rollout_episodes\(pcl_handle\* h, const int32_t\* d_actions, '
                   r'int steps,\s+const pcl_outputs\* out, const pcl_rollout_rec\* rec,\s+'
                   r'const pcl_episode_rec\* ep, void\* stream\);', header)
  assert int(re.search(r'#define PCL_ABI_VERSION (\d+)', header).group(1)) == 3


def _handle(bind=True):
  lib = _lib.load()
  spec = _lib.Spec()
  spec.abi_version, spec.program = _lib.ABI_VERSION, _lib.PROG_NONE
  spec.rows, spec.cols, spec.pitch = 16, 16, 16
  spec.n_sprites, spec.n_drapes = 2, 2
  h = C.c_void_p()
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(h)) == _lib.OK
  if bind:
    assert lib.pcl_bind_state(h, C.byref(boundary_sweep._full_state())) == _lib.OK
  return lib, h


def _outputs():
  return _lib.Outputs(FAKE, FAKE, FAKE, FAKE, FAKE, FAKE)


def _call(lib, h, ep, steps=3, rec=None):
  return lib.pcl_rollout_episodes(h, FAKE, steps, C.byref(_outputs()),
                                  None if rec is None else C.byref(rec),
                                  None if ep is None else C.byref(ep), None)


def test_bind_episodes_refusals():
  lib, h = _handle(bind=False)
  try:
    assert lib.pcl_bind_episodes(None, FAKE) == _lib.ERR_INVALID
    assert lib.pcl_bind_episodes(None, None) == _lib.ERR_INVALID
    for off in (1, 2, 4, 7):
      assert lib.pcl_bind_episodes(h, FAKE + off) == _lib.ERR_INVALID, off
    assert lib.pcl_bind_episodes(h, FAKE) == _lib.OK      # before pcl_bind_state too
    assert lib.pcl_bind_episodes(h, None) == _lib.OK      # tracking off
    assert lib.pcl_bind_episodes(h, FAKE + 8) == _lib.OK
  finally:
    lib.pcl_destroy(h)


def test_rollout_episodes_refusals():
  lib, h = _handle()
  try:
    # kept arrays on a handle with no bound returns
    for ep in (_lib.EpisodeRec(FAKE, None), _lib.EpisodeRec(None, FAKE),
               _lib.EpisodeRec(FAKE, FAKE)):
      assert _call(lib, h, ep) == _lib.ERR_INVALID
      assert _call(lib, h, ep, steps=0) == _lib.ERR_INVALID
    assert _call(lib, h, _lib.EpisodeRec(), steps=0) == _lib.OK     # nothing kept, no step
    assert _call(lib, h, None, steps=0) == _lib.OK
    assert lib.pcl_bind_episodes(h, FAKE) == _lib.OK
    for ep in (_lib.EpisodeRec(FAKE + 4, None), _lib.EpisodeRec(FAKE + 1, FAKE),
               _lib.EpisodeRec(None, FAKE + 2), _lib.EpisodeRec(FAKE, FAKE + 3)):
      assert _call(lib, h, ep) == _lib.ERR_INVALID
    # the common refusals come first, as pcl_rollout's
    assert lib.pcl_rollout_episodes(None, FAKE, 1, C.byref(_outputs()), None,
                                    C.byref(_lib.EpisodeRec(FAKE, FAKE)), None) == \
        _lib.ERR_INVALID
    assert _call(lib, h, _lib.EpisodeRec(FAKE, FAKE), steps=-1) == _lib.ERR_INVALID
    assert _call(lib, h, _lib.EpisodeRec(FAKE, FAKE), steps=0) == _lib.OK
    assert lib.pcl_bind_episodes(h, None) == _lib.OK
    assert _call(lib, h, _lib.EpisodeRec(FAKE, FAKE), steps=0) == _lib.ERR_INVALID
  finally:
    lib.pcl_destroy(h)


def test_the_binding_survives_bind_state():
  lib, h = _handle()
  try:
    assert lib.pcl_bind_episodes(h, FAKE) == _lib.OK
    assert lib.pcl_bind_state(h, C.byref(boundary_sweep._full_state())) == _lib.OK
    assert _call(lib, h, _lib.EpisodeRec(FAKE, FAKE), steps=0) == _lib.OK
  finally:
    lib.pcl_destroy(h)


def test_unbound_handle_is_refused_first():
  lib, h = _handle(bind=False)
  try:
    assert lib.pcl_bind_episodes(h, FAKE) == _lib.OK
    assert _call(lib, h, _lib.EpisodeRec(FAKE, FAKE)) == _lib.ERR_UNBOUND
  finally:
    lib.pcl_destroy(h)


@pytest.mark.parametrize('bad', [1, 0, None, 'yes', np.bool_(True)])
def test_facade_refuses_a_non_bool_before_cuda(bad):
  from pycolab_b200 import batched
  from pycolab_b200.games.classics import four_rooms
  with pytest.raises(TypeError, match='track_episodes'):
    batched.BatchedEngine([four_rooms.make_game()], batch=2, track_episodes=bad)


def test_shard_engine_forwards_track_episodes():
  from pycolab_b200 import dist
  from pycolab_b200.games.classics import four_rooms
  with pytest.raises(TypeError, match='track_episodes'):
    dist.make_shard_engine([four_rooms.make_game()], 4, 1, 2, 0, track_episodes='on')


def _facade_engine(track):
  """A BatchedEngine shell that reaches no device: what rollout()'s checks read."""
  import torch
  from pycolab_b200 import batched
  eng = batched.BatchedEngine.__new__(batched.BatchedEngine)
  eng.batch, eng.actions_per_env, eng._showtime = 3, 1, True
  eng.device = torch.device('cpu')
  eng.episode_return = torch.zeros(3, dtype=torch.float64) if track else None
  return eng


def test_facade_refuses_episodes_on_a_non_tracking_engine():
  from pycolab_b200 import batched
  eng = _facade_engine(track=False)
  with pytest.raises(ValueError, match='track_episodes=True'):
    eng.new_episodes(4)


def test_facade_makes_episodes_of_the_rollout_shape():
  import torch
  from pycolab_b200 import batched
  ep = _facade_engine(track=True).new_episodes(4)
  assert isinstance(ep, batched.Episodes)
  assert ep.episode_return.shape == (4, 3) and ep.episode_return.dtype == torch.float64
  assert ep.episode_length.shape == (4, 3) and ep.episode_length.dtype == torch.int32
  assert batched.Episodes.__slots__ == ('episode_return', 'episode_length')
  assert 'episode_return' not in batched.Trajectory.__slots__


# ---- the host reference ---------------------------------------------------------------

def test_reference_restart_mid_run_and_frame_zero_reward():
  # env 0: showtime pays 3, two steps pay 1 and None, restart pays 5, then 2
  reward = np.array([[3, 0], [1, 7], [0, 0], [5, 4], [2, 0]])
  has = np.array([[1, 0], [1, 1], [0, 1], [1, 1], [1, 0]])
  frame = np.array([[0, 0], [1, 1], [2, 2], [0, 3], [1, 4]])
  got = ref.returns(reward, has, frame)
  assert got[:, 0].tolist() == [3.0, 4.0, 4.0, 5.0, 7.0]
  assert got[:, 1].tolist() == [0.0, 7.0, 7.0, 11.0, 11.0]


def test_reference_truncation_keeps_the_sum_to_the_cut():
  # a time limit of 2: done 2 at frame 2, the next step restarts at frame 0
  reward = np.array([[0], [1], [1], [0], [1]])
  frame = np.array([[0], [1], [2], [0], [1]])
  got = ref.returns(reward, np.ones_like(reward), frame)
  assert got[:, 0].tolist() == [0.0, 1.0, 2.0, 0.0, 1.0]


def test_reference_frozen_envs_keep_their_return():
  reward = np.array([[0, 0], [2, 1], [9, 9], [9, 9]])
  frame = np.array([[0, 0], [1, 1], [1, 2], [1, 3]])
  ran = np.array([[1, 1], [1, 1], [0, 1], [0, 1]], bool)
  got = ref.returns(reward, np.ones_like(reward), frame, ran=ran, start=[-1.0, -1.0])
  assert got[:, 0].tolist() == [0.0, 2.0, 2.0, 2.0]
  assert got[:, 1].tolist() == [0.0, 1.0, 10.0, 19.0]
  # an env that never (re)starts keeps what the buffer held
  got = ref.returns(reward[1:], np.ones((3, 2)), frame[1:], ran=ran[1:] * 0, start=[4.5, 0.0])
  assert got[:, 0].tolist() == [4.5] * 3


def test_reference_float_sums_are_in_step_order():
  # 0.1 + 0.2 + 0.3 in order is not 0.6, nor what cumsum-minus-prefix gives
  reward = np.array([[0.0], [0.1], [0.2], [0.3], [1e16], [1.0], [-1e16]])
  frame = np.arange(7).reshape(7, 1)
  got = ref.returns(reward, np.ones((7, 1)), frame)
  want, acc = [], 0.0
  for t in range(7):
    acc = reward[t, 0] if t == 0 else acc + reward[t, 0]
    want.append(acc)
  assert ref.same_bits(got[:, 0], want)
  assert got[3, 0] != 0.6
  assert got[6, 0] == 0.0 and got[5, 0] - 1e16 == 0.0    # 1e16 + 1.0 rounds the 1.0 away


def test_same_bits_tells_signed_zeros_apart():
  assert ref.same_bits([0.0, 1.5], [0.0, 1.5])
  assert not ref.same_bits([0.0], [-0.0])
  assert not ref.same_bits([1.0], [1.0, 1.0])
