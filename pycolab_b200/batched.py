"""`BatchedEngine`: B independent pycolab environments stepped in lockstep on one GPU.

The batched counterpart of the reference's one-`Engine`-per-env loop
(engine.py:520-639): `its_showtime()` / `play(actions)` keep their meaning,
vectorised over the env axis.  State lives in HBM as a struct-of-arrays
(include/pcl.h `pcl_state`); PyTorch is used only to own the device buffers
and the stream.  Every step is ONE fused CUDA kernel launched through the
C ABI (`pcl_step`); there is no CPU path.
"""

import ctypes as C
import numbers
import operator
import random

import numpy as np

from pycolab_b200 import _lib
from pycolab_b200 import lowering
from pycolab_b200.errors import NotLoweredError


def _torch():
  import torch
  return torch


def _check_crop(status, what, handle, crop_spec):
  """`_lib.check` for a cropper entry point: a window or tracking list the device does
  not serve (PCL_ERR_UNSUPPORTED) raises NotLoweredError."""
  if status == _lib.ERR_UNSUPPORTED:
    raise NotLoweredError(
        '%s: the device does not serve this cropper (%dx%d window, at most %d cells; '
        'tracking list %s; drapes are tracked by crop() on boards up to 128x128 only)' % (
            what, crop_spec.rows, crop_spec.cols, _lib.MAX_CROP_CELLS, list(crop_spec.track)))
  _lib.check(status, what, handle)


def _time_limit(n):
  """The pcl_set_time_limit value of a `time_limit` argument: None or 0 is no limit."""
  if n is None:
    return 0
  if isinstance(n, bool) or not isinstance(n, numbers.Integral):
    raise TypeError('time_limit is None or an int number of steps, got %r' % (n,))
  if not 0 <= n < 2 ** 31:
    raise ValueError('time_limit is None, 0 (no limit) or a number of steps below 2**31, '
                     'got %d' % n)
  return int(n)


def _mt_state(stream, seed):
  """u32 [625]: the MT19937 words (624 key words + position) of a generator seeded with
  `seed`: Python's random.Random ('python') or NumPy's RandomState ('numpy')."""
  if stream == 'python':
    return np.array(random.Random(seed).getstate()[1], dtype=np.uint32)
  _, key, pos, _, _ = np.random.RandomState(seed).get_state()
  return np.append(key, pos).astype(np.uint32)


SEED_LIMIT = 2 ** 32             # pcl_seed_rng takes seeds in [0, SEED_LIMIT)


def _device_seeded(rng_seed, env_offset, batch):
  """Does the constructor seed its generators on the device (pcl_seed_rng)?  Only when every
  env's seed rng_seed + env_offset + e is an int in [0, 2**32), where the kernel writes the
  words `_mt_state` would.  Other seeds keep the host words: a game that draws from Python's
  `random` only takes any int there, and NumPy raises for them as it always has."""
  if not (isinstance(rng_seed, numbers.Integral) and isinstance(env_offset, numbers.Integral)):
    return False
  first = int(rng_seed) + int(env_offset)
  return 0 <= first and first + int(batch) <= SEED_LIMIT


class StepResult(object):
  """(board, reward, has_reward, discount, done) of one batched step.

  board: u8 [B, rows, cols] view into the engine-owned output buffer (valid
  until the next step — copy to keep, as upstream rendering.py:55-63).
  reward: i32 [B] (f64 [B] for games whose rewards are not integers, e.g. t_maze) with
  has_reward u8 [B] == 0 where the reference returns None.
  discount: f32 [B].  done: u8 [B] (Engine.game_over): 0 running, 1 ended by the game, 2
  (_lib.DONE_TIME_LIMIT) ended by the engine's time limit, with the step's own reward and
  discount.
  """
  __slots__ = ('board', 'reward', 'has_reward', 'discount', 'done')

  def __init__(self, board, reward, has_reward, discount, done):
    self.board, self.reward, self.has_reward = board, reward, has_reward
    self.discount, self.done = discount, done

  def __iter__(self):            # (observation, reward, discount) like Engine.play
    return iter((self.board, self.reward, self.discount))


class Trajectory(object):
  """What `BatchedEngine.rollout` kept of T steps, each a [T, B, ...] device tensor.

  reward: i32 [T, B] (f64 for games whose rewards are not integers, as `reward`);
  has_reward, done: u8 [T, B]; discount: f32 [T, B].  Slot t holds what play() leaves in
  the engine's outputs after step t; done is 0 running, 1 ended by the game, 2 ended by the
  time limit (a truncation: the discount is the game's).  An env frozen at step t (auto_reset
  off) holds done 1, has_reward 0, reward 0 and discount 0.0.  view: the observer's result of
  every step, [T] + what to_feature_array / to_array / repaint return for one step, or None.
  attached: u8 [T, B, rows, cols], the attached cropper's view of every step, or None.
  unknown: i32 [1] for an ObservationToArray observer, 1 when a step met a character
  outside its mapping; else None.
  Pass the Trajectory as `out=` to a later rollout of the same shape to reuse its buffers.
  """
  __slots__ = ('reward', 'has_reward', 'discount', 'done', 'view', 'attached', 'unknown')

  def __init__(self, reward, has_reward, discount, done, view, attached, unknown):
    self.reward, self.has_reward, self.discount, self.done = reward, has_reward, discount, done
    self.view, self.attached, self.unknown = view, attached, unknown


class Episodes(object):
  """The episode returns and lengths `BatchedEngine.rollout(..., episodes=)` kept of T
  steps, each a [T, B] device tensor.

  episode_return: f64 [T, B], the env's episode return after step t (the engine's
  `episode_return` then).  episode_length: i32 [T, B], the env's frame after step t: the
  number of play()s since its (re)start.  At a step whose done is nonzero they are the
  finished episode's return and length, so with `traj` the rollout's Trajectory

      finished_returns = ep.episode_return[traj.done > 0]
      finished_lengths = ep.episode_length[traj.done > 0]

  are what a training loop logs.  An env frozen at step t (auto_reset off) holds 0.0 and 0.
  Make one with `BatchedEngine.new_episodes(T)`, and pass it again to reuse its buffers.
  """
  __slots__ = ('episode_return', 'episode_length')

  def __init__(self, episode_return, episode_length):
    self.episode_return, self.episode_length = episode_return, episode_length


class BatchedEngine(object):

  def __init__(self, games, batch=None, device=0, auto_reset=True, rng_seed=0,
               env_offset=0, rng_states=None, share_levels=True, time_limit=None,
               track_episodes=False):
    """games: list of lowered games (`lowering.LoweredGame`) or set-up `Engine`s.
    Env e uses games[e % len(games)]; with a single game the static level data
    (backdrop, immutable patterns, reset templates) is shared by all envs.
    env_offset: global index of this shard's env 0 (per-env RNG streams are
    seeded rng_seed + global env index — NumPy RandomState(seed) or, for games that
    draw from Python's `random`, random.Random(seed); written on the device by pcl_seed_rng
    when every such seed lies in [0, 2**32), else on the host); rng_states: explicit u32 [B, 625]
    (False: bind no RNG, for programs that can take their draws from the templates)
    MT19937 states (624 key words + position) instead of seeds.
    share_levels=False stores the static level data once PER ENV instead of once
    per level (the reference's layout: every Engine owns its backdrop).
    time_limit: see set_time_limit; None (the default) or 0 is no limit.
    track_episodes: keep each env's episode return on the device (`episode_return`)."""
    limit = _time_limit(time_limit)
    if not isinstance(track_episodes, bool):
      raise TypeError('track_episodes is True or False, got %r' % (track_episodes,))
    torch = _torch()
    self._lib = _lib.load()
    if not torch.cuda.is_available():
      raise _lib.PclLibraryError('CUDA device required: pycolab_b200 has no CPU path')
    games = [g if isinstance(g, lowering.LoweredGame) else lowering.lower(g)
             for g in (games if isinstance(games, (list, tuple)) else [games])]
    sig = games[0].signature()
    for g in games[1:]:
      if g.signature() != sig:
        raise ValueError('all games of one BatchedEngine must share one structure')
    self.game = g0 = games[0]
    self.batch = B = int(batch if batch is not None else len(games))
    self.device = torch.device('cuda', device)
    self.auto_reset = bool(auto_reset)
    self.rows, self.cols, self.pitch = g0.rows, g0.cols, g0.pitch
    self.sprite_chars, self.drape_chars = g0.sprite_chars, g0.drape_chars
    # object chars (LoweredGame.object_chars) may differ between the levels of one handle
    self.object_chars = ''.join(sorted(set(''.join(g.object_chars for g in games))))
    self.chars = ''.join(sorted(set(g0.sprite_chars + g0.drape_chars + g0.backdrop_chars +
                                    self.object_chars)))
    n = len(games)
    shared = (n == 1)
    dev = self.device

    def tiled(arrays, dtype):
      """Static data: ONE copy per level ([n_levels, ...]); envs find theirs
      through the level index (pcl_state.d_level), or share the single copy."""
      stacked = np.stack([np.ascontiguousarray(a).astype(dtype) for a in arrays])
      return torch.from_numpy(stacked).to(dev)

    def per_env(arrays, dtype):
      stacked = np.stack([np.ascontiguousarray(a).astype(dtype) for a in arrays])
      t = torch.from_numpy(stacked).to(dev)
      reps = (B + n - 1) // n
      return t.repeat((reps,) + (1,) * (t.dim() - 1))[:B].contiguous()

    def bstride(t):
      return 0 if t.shape[0] == 1 else t[0].numel()

    if not share_levels:
      tiled, shared = per_env, True     # every array env-indexed, no level table

    self._keep = []             # every tensor the handle points at
    st = _lib.State()
    self.level = None           # i32 [B]: which level each env plays
    if not shared:
      self.level = (torch.arange(B, dtype=torch.int32, device=dev) % n).contiguous()
      st.d_level = self.level.data_ptr()
    self.backdrop = tiled([g.backdrop for g in games], np.uint8)
    st.d_backdrop, st.backdrop_bstride = self.backdrop.data_ptr(), bstride(self.backdrop)
    self.patterns, self.bits = {}, {}
    self._keep_bits_init = {}
    draws = g0.needs_rng and rng_states is not False
    for d in sorted(g0.patterns):
      arrays = [g.patterns[d].view(np.int32) for g in games]
      if g0.pattern_mutable[d]:
        # a pattern the device redraws at every restart resets from its un-drawn template
        init = tiled([g.pattern_redraw[d].view(np.int32) for g in games]
                     if draws and d in g0.pattern_redraw else arrays, np.int32)
        live = per_env(arrays, np.int32)
        st.d_pattern_init[d], st.pattern_init_bstride[d] = init.data_ptr(), bstride(init)
        self._keep.append(init)
      else:
        live = tiled(arrays, np.int32)
      self.patterns[d] = live
      st.d_pattern[d] = live.data_ptr()
      st.pattern_bstride[d] = bstride(live) if not g0.pattern_mutable[d] else live[0].numel()
    for d in sorted(g0.bits):
      arrays = [g.bits[d].view(np.int32) for g in games]
      init = tiled(arrays, np.int32)
      live = per_env(arrays, np.int32)
      self.bits[d] = live
      self._keep.append(init)
      self._keep_bits_init[d] = init
      st.d_bits[d], st.bits_bstride[d] = live.data_ptr(), live[0].numel()
      st.d_bits_init[d], st.bits_init_bstride[d] = init.data_ptr(), bstride(init)
    self.sprites = per_env([g.sprites for g in games], np.int32)
    self.drapes = per_env([g.drapes for g in games], np.int32)
    self.plot = per_env([g.plot for g in games], np.int32)
    # Live records start "game over" so the first pcl_reset builds every env.
    self._sprites_init = tiled([g.sprites for g in games], np.int32)
    self._drapes_init = tiled([g.drapes for g in games], np.int32)
    self._plot_init = tiled([g.plot for g in games], np.int32)
    st.d_sprites, st.d_sprites_init = self.sprites.data_ptr(), self._sprites_init.data_ptr()
    st.sprites_init_bstride = bstride(self._sprites_init)
    st.d_drapes, st.d_drapes_init = self.drapes.data_ptr(), self._drapes_init.data_ptr()
    st.drapes_init_bstride = bstride(self._drapes_init)
    st.d_plot, st.d_plot_init = self.plot.data_ptr(), self._plot_init.data_ptr()
    st.plot_init_bstride = bstride(self._plot_init)
    self.z_order = None
    if g0.dynamic_z:
      zs = [np.frombuffer(g.z_order.encode('ascii'), dtype=np.uint8) for g in games]
      self.z_order = per_env(zs, np.uint8)
      self._z_init = tiled(zs, np.uint8)
      st.d_z_order, st.d_z_order_init = self.z_order.data_ptr(), self._z_init.data_ptr()
      st.z_order_init_bstride = bstride(self._z_init)
    self.groups = None          # scrolling groups >= 1 (group 0 is in the plot record)
    if len(g0.scroll_groups) > 1:
      self.groups = per_env([g.group_records for g in games], np.int32)
      self._groups_init = tiled([g.group_records for g in games], np.int32)
      st.d_groups, st.d_groups_init = self.groups.data_ptr(), self._groups_init.data_ptr()
      st.groups_init_bstride = bstride(self._groups_init)
    self.actions_per_env = g0.actions_per_env
    self.env_offset = env_offset
    self.rng = None             # u32 [B, slots * 625] as int32: each env's generator words
    seed_on_device = False
    if draws:
      slots = len(g0.rng_streams)
      if rng_states is not None:
        states = np.ascontiguousarray(rng_states, dtype=np.uint32).reshape(
            B, slots * _lib.MT_WORDS)
        self.rng = torch.from_numpy(states.view(np.int32)).to(dev)
      elif _device_seeded(rng_seed, env_offset, B):
        seed_on_device = True     # written by pcl_seed_rng once the state is bound
        self.rng = torch.empty((B, slots * _lib.MT_WORDS), dtype=torch.int32, device=dev)
      else:
        states = np.stack([np.concatenate([_mt_state(stream, rng_seed + env_offset + e)
                                           for stream in g0.rng_streams]) for e in range(B)])
        self.rng = torch.from_numpy(states.view(np.int32)).to(dev)
      st.d_rng = self.rng.data_ptr()
      self._seed_kinds = (C.c_int32 * slots)(*[
          _lib.SEED_PYTHON if stream == 'python' else _lib.SEED_NUMPY
          for stream in g0.rng_streams])
    self._state = st

    # Outputs.
    self._board = torch.zeros((B, self.rows, self.pitch), dtype=torch.uint8, device=dev)
    self.reward = torch.zeros((B,), dtype=torch.int32, device=dev)
    self.has_reward = torch.zeros((B,), dtype=torch.uint8, device=dev)
    self.discount = torch.ones((B,), dtype=torch.float32, device=dev)
    self.done = torch.zeros((B,), dtype=torch.uint8, device=dev)
    self._out = _lib.Outputs(self._board.data_ptr(), self.reward.data_ptr(),
                             self.has_reward.data_ptr(), self.discount.data_ptr(),
                             self.done.data_ptr())
    if g0.float_reward:
      # the kernel writes the float64 sum (pcl_outputs.d_reward_f64) and leaves d_reward alone
      self._reward_i32 = self.reward
      self.reward = torch.zeros((B,), dtype=torch.float64, device=dev)
      self._out.d_reward_f64 = self.reward.data_ptr()
    self._actions = torch.zeros((B * self.actions_per_env,), dtype=torch.int32, device=dev)
    self._host = None           # pinned staging for play_host() / play_host_async(), per slot
    self._slot_shape = {}
    self._crop_dev = None
    self._crop_out = None
    self._attached = None       # attach_cropper: (spec, state, out, runs inside the step kernel)
    self._tables = None         # rollout: id(observer), over a window -> its device tables

    self._spec = g0.make_spec(self.auto_reset)
    handle = C.c_void_p()
    _lib.check(self._lib.pcl_create(C.byref(self._spec), B, self.device.index,
                                    C.byref(handle)), 'pcl_create')
    self._h = handle
    _lib.check(self._lib.pcl_bind_state(self._h, C.byref(self._state)), 'pcl_bind_state')
    if seed_on_device:
      self._seed(None, self._seed_tensor(int(rng_seed)))
    if g0.code is not None:       # the compiled program's bytecode, shared by every level
      code = np.ascontiguousarray(g0.code, dtype=np.int32)
      _lib.check(self._lib.pcl_bind_code(self._h, code.ctypes.data, len(code)), 'pcl_bind_code')
    self.backdrop_live = None   # u8 [B, rows, pitch]: a compiled Backdrop's curtains as they are now
    if g0.program == _lib.PROG_COMPILED and g0.program_arg[4]:
      self.backdrop_live = per_env([g.backdrop for g in games], np.uint8)
      _lib.check(self._lib.pcl_bind_backdrop(self._h, self.backdrop_live.data_ptr()),
                 'pcl_bind_backdrop')
    self.time_limit = 0
    self.set_time_limit(limit)
    # f64 [B]: each env's episode return, updated on the device by every step and reset
    # (pcl_bind_episodes): the sum of the rewards since the env's (re)start, its reset frame's
    # included, added in step order as `ret = r if frame == 0 else ret + r` does over the
    # engine's own reward and frame.  At a step with done != 0 it is the finished episode's
    # return, and the env's plot frame its length.  None unless track_episodes.
    self.episode_return = None
    if track_episodes:
      self.episode_return = torch.zeros((B,), dtype=torch.float64, device=dev)
      _lib.check(self._lib.pcl_bind_episodes(self._h, self.episode_return.data_ptr()),
                 'pcl_bind_episodes')
    self._showtime = False

  def set_time_limit(self, n):
    """End every episode after n steps (pcl_set_time_limit); None or 0: no limit.

    A step that leaves an env at frame n or later (n play()s after its its_showtime() or
    restart frame) reports done 2 (_lib.DONE_TIME_LIMIT) unless the game ended the episode
    in that step, which stays done 1.  Reward, discount and board are the step's own.  The
    next step restarts the env under auto_reset and freezes it otherwise, as after any
    ending; reset(mask) starts an env's count afresh.  Upstream pycolab has no time limit:
    with none set the engine behaves exactly as without this call.  Applies from the next
    step; a CUDA graph captured earlier keeps the limit it was captured with."""
    limit = _time_limit(n)
    _lib.check(self._lib.pcl_set_time_limit(self._h, limit), 'pcl_set_time_limit')
    self.time_limit = limit

  # ---------------------------------------------------------------- running
  def _stream(self):
    return C.c_void_p(_torch().cuda.current_stream(self.device).cuda_stream)

  @property
  def board(self):
    """u8 [B, rows, cols] view of the last rendered boards."""
    return self._board[:, :, :self.cols]

  def _result(self):
    return StepResult(self.board, self.reward, self.has_reward, self.discount, self.done)

  def its_showtime(self):
    """Engine.its_showtime() for every env (engine.py:520-581)."""
    if self._showtime:
      raise RuntimeError('its_showtime should not be called after its_showtime() has '
                         'been called')
    self._showtime = True
    _lib.check(self._lib.pcl_reset(self._h, None, C.byref(self._out), self._stream()),
               'pcl_reset', self._h)
    self._after_step()
    return self._result()

  def reset(self, env_mask=None, seeds=None):
    """Rebuild the selected envs (u8/bool [B] device tensor; None = all) and run
    their its_showtime() frame; other envs are untouched.

    seeds: first seed each selected env's generators as a fresh generator with that seed
    would be, Gymnasium's reset(seed=...) per env: an int s (env e gets s + env_offset + e,
    the constructor's rng_seed rule, so shards agree) or ints [B] (a sequence or tensor),
    each in [0, 2**32).  A Python-`random` slot gets random.Random(seed)'s words, a NumPy
    slot RandomState(seed)'s, so the env's episode is the one an engine built with that
    seed plays.  Two launches on the current stream (pcl_seed_rng, then pcl_reset), so a
    CUDA graph may hold them; the range of a CUDA tensor's seeds is not checked while the
    stream is being captured.  Draws the game made when it was built (the reset templates)
    are not redrawn."""
    d_seeds = None if seeds is None else self._seed_tensor(seeds)
    self._showtime = True
    mask = None
    if env_mask is not None:
      mask = env_mask.to(device=self.device, dtype=_torch().uint8).contiguous()
    if d_seeds is not None:
      self._seed(mask, d_seeds)
    _lib.check(self._lib.pcl_reset(self._h, None if mask is None else mask.data_ptr(),
                                   C.byref(self._out), self._stream()), 'pcl_reset', self._h)
    self._after_step()
    return self._result()

  def _seed_tensor(self, seeds):
    """The u32 [B] seeds of `reset(seeds=)` as an int32 device tensor of the same bits."""
    torch = _torch()
    if self.rng is None:
      raise ValueError('seeds= needs an engine whose game draws from random generators on the '
                       'device; this one has none (the game draws nothing, rng_states=False, '
                       'or its levels are generated on the host)')
    B = self.batch
    if isinstance(seeds, numbers.Integral) and not isinstance(seeds, (bool, np.bool_)):
      first = int(seeds) + int(self.env_offset)
      if not (0 <= first and first + B <= SEED_LIMIT):
        raise ValueError('seed %d gives env seeds %d .. %d (env_offset %d); each must lie in '
                         '[0, 2**32)' % (int(seeds), first, first + B - 1, self.env_offset))
      t = torch.arange(first, first + B, dtype=torch.int64, device=self.device)
    else:
      if torch.is_tensor(seeds):
        t = seeds
      else:
        if isinstance(seeds, np.ndarray) and seeds.ndim != 1:
          raise ValueError('expected %d seeds, one per env, got shape %s' % (B, seeds.shape))
        try:
          vals = [operator.index(s) for s in seeds]
        except TypeError:
          raise TypeError('seeds is an int or a [B] sequence or tensor of ints, got %r' % (
              seeds,))
        if len(vals) != B:
          raise ValueError('expected %d seeds, one per env, got %d' % (B, len(vals)))
        if vals and (min(vals) < 0 or max(vals) >= SEED_LIMIT):
          raise ValueError('each seed must lie in [0, 2**32)')
        t = torch.tensor(vals, dtype=torch.int64)
      if t.dtype == torch.bool or t.dtype.is_floating_point or t.dtype.is_complex:
        raise TypeError('seeds is an int or a [B] sequence or tensor of ints, got %s' % t.dtype)
      if tuple(t.shape) != (B,):
        raise ValueError('expected %d seeds, one per env, got shape %s' % (B, tuple(t.shape)))
      t = t.to(device=self.device, dtype=torch.int64)
      if B and not (t.is_cuda and torch.cuda.is_current_stream_capturing()):
        if bool(((t < 0) | (t >= SEED_LIMIT)).any()):
          raise ValueError('each seed must lie in [0, 2**32)')
    # the low 32 bits, as an int32 holds them
    return torch.where(t >= 2 ** 31, t - SEED_LIMIT, t).to(torch.int32).contiguous()

  def _seed(self, mask, d_seeds):
    """pcl_seed_rng of the envs `mask` selects (None = all) on the current stream."""
    _lib.check(self._lib.pcl_seed_rng(self._h, None if mask is None else mask.data_ptr(),
                                      d_seeds.data_ptr(), self._seed_kinds,
                                      len(self._seed_kinds), self._stream()),
               'pcl_seed_rng', self._h)

  def play(self, actions):
    """Engine.play(actions) for every env (engine.py:583-639).

    actions: int32 [B] device tensor (or anything torch.as_tensor accepts).
    With auto_reset, an env that was game-over is rebuilt instead and its
    action is ignored; without it such envs stay frozen (upstream raises)."""
    if not self._showtime:
      raise RuntimeError('play() cannot be called until the Engine is placed in "play '
                         'mode" via the its_showtime() method.')
    torch = _torch()
    if not (torch.is_tensor(actions) and actions.is_cuda and
            actions.dtype == torch.int32 and actions.is_contiguous()):
      actions = torch.as_tensor(actions, dtype=torch.int32).to(self.device).contiguous()
    if actions.numel() != self.batch * self.actions_per_env:
      raise ValueError('expected %d action words, got %d' % (
          self.batch * self.actions_per_env, actions.numel()))
    _lib.check(self._lib.pcl_step(self._h, actions.data_ptr(), C.byref(self._out),
                                  self._stream()), 'pcl_step', self._h)
    self._after_step()
    return self._result()

  def run(self, actions):
    """T back-to-back steps; actions int32 [T, B] on the device."""
    torch = _torch()
    assert actions.is_cuda and actions.dtype == torch.int32 and actions.is_contiguous()
    assert actions.dim() >= 2 and actions[0].numel() == self.batch * self.actions_per_env
    _lib.check(self._lib.pcl_run(self._h, actions.data_ptr(), int(actions.shape[0]),
                                 C.byref(self._out), self._stream()), 'pcl_run', self._h)
    return self._result()

  def new_episodes(self, T):
    """An `Episodes` of T steps for `rollout(..., episodes=)` on this engine."""
    torch = _torch()
    if self.episode_return is None:
      raise ValueError('episodes need an engine made with track_episodes=True')
    T = int(T)
    return Episodes(torch.zeros((T, self.batch), dtype=torch.float64, device=self.device),
                    torch.zeros((T, self.batch), dtype=torch.int32, device=self.device))

  def rollout(self, actions, observer=None, crop_spec=None, state=None, keep_attached=False,
              out=None, episodes=None):
    """T steps from one C call (`pcl_rollout`), keeping every step's outputs.

    actions: int32 [T, B] or [T, B, actions_per_env] on the device.  Each step is play(),
    then the attached cropper, then `observer` (a `rendering.ObservationToFeatureArray`,
    `ObservationToArray` or `ObservationCharacterRepainter`) over the board or, with
    `crop_spec`, over that cropper's window (its corner in `state`), as
    to_feature_array / to_array / repaint would run it.  Returns a `Trajectory`; with
    keep_attached, it also holds the attached cropper's view of every step.  Afterwards
    the engine's outputs and the attached view are step T-1's, as after T play()s.

    An ObservationToArray raises RuntimeError, as to_array does, when any step met a
    character outside its mapping; the flag is read once per call, and not at all while
    the stream is being captured (read `Trajectory.unknown` then).  `out`: a Trajectory
    of an earlier rollout of the same shape, whose buffers are reused, so that a captured
    rollout replays into fixed memory.

    `episodes`: an `Episodes` (new_episodes(T)) that also keeps every step's episode return
    and length, on an engine made with track_episodes=True; `ep.episode_return[traj.done >
    0]` and `ep.episode_length[traj.done > 0]` are then the episodes that finished in the
    rollout.  Afterwards `episode_return` is step T-1's, as after T play()s."""
    torch = _torch()
    if not self._showtime:
      raise RuntimeError('rollout() cannot be called until the Engine is placed in "play '
                         'mode" via the its_showtime() method.')
    if not (torch.is_tensor(actions) and actions.is_cuda and actions.dtype == torch.int32 and
            actions.is_contiguous()):
      raise TypeError('rollout actions are a contiguous int32 CUDA tensor [T, B(, words)]')
    if actions.dim() < 2 or int(np.prod(actions.shape[1:])) != self.batch * self.actions_per_env:
      raise ValueError('expected [T, %d] actions of %d words per env, got %s' % (
          self.batch, self.actions_per_env, tuple(actions.shape)))
    T, B = int(actions.shape[0]), self.batch
    att = self._attached
    if keep_attached and att is None:
      raise ValueError('keep_attached needs a cropper attached with attach_cropper()')
    obs = self._rollout_observer(observer, crop_spec)
    crop = crop_spec if obs is not None else None
    rows, cols = (crop.rows, crop.cols) if crop is not None else (self.rows, self.cols)
    dev = self.device
    want = dict(reward=((T, B), self.reward.dtype), has_reward=((T, B), torch.uint8),
                discount=((T, B), torch.float32), done=((T, B), torch.uint8))
    if keep_attached:
      want['attached'] = ((T, B, att[0].rows, att[0].cols), torch.uint8)
    if obs is not None:
      base = [obs['depth'], rows, cols] if obs['is_3d'] else [rows, cols]
      perm = obs['permute'] if obs['permute'] is not None else range(len(base))
      want['view'] = (tuple([T, B] + [base[i] for i in perm]), obs['dtype'])
      if obs['check']:
        want['unknown'] = ((1,), torch.int32)
    ep_rec = None
    if episodes is not None:
      if self.episode_return is None:
        raise ValueError('episodes= needs an engine made with track_episodes=True')
      if not isinstance(episodes, Episodes):
        raise TypeError('episodes= is an Episodes (new_episodes(T)), not %r' % (
            type(episodes).__name__,))
      for name, dtype in (('episode_return', torch.float64), ('episode_length', torch.int32)):
        got = getattr(episodes, name)
        if (not torch.is_tensor(got) or tuple(got.shape) != (T, B) or got.dtype != dtype or
            got.device != dev or not got.is_contiguous()):
          raise ValueError('episodes.%s is not a contiguous %s %s on %s' % (
              name, dtype, (T, B), dev))
      ep_rec = _lib.EpisodeRec(episodes.episode_return.data_ptr() if T else None,
                               episodes.episode_length.data_ptr() if T else None)
    traj = out if out is not None else Trajectory(*[None] * 7)
    for name in Trajectory.__slots__:
      got = getattr(traj, name)
      if name not in want:
        if out is None:
          continue
        if got is not None:
          raise ValueError('out= holds a %s this rollout does not produce' % name)
      elif out is None:
        setattr(traj, name, torch.empty(want[name][0], dtype=want[name][1], device=dev))
      elif got is None or tuple(got.shape) != want[name][0] or got.dtype != want[name][1]:
        raise ValueError('out=.%s is not %s %s' % (name, want[name][1], want[name][0]))
    rec = _lib.RolloutRec()
    if self.game.float_reward:
      rec.d_reward_f64 = traj.reward.data_ptr()
    else:
      rec.d_reward = traj.reward.data_ptr()
    rec.d_has_reward, rec.d_done = traj.has_reward.data_ptr(), traj.done.data_ptr()
    rec.d_discount = traj.discount.data_ptr()
    if keep_attached:
      rec.d_attached = traj.attached.data_ptr()
    if att is not None and not att[3]:          # the cropper that _after_step runs
      rec.crop = C.pointer(att[0])
      rec.d_crop_state, rec.d_crop = att[1].data_ptr(), att[2].data_ptr()
    view = None
    if obs is not None:
      spec = obs['spec'](traj.view)
      rec.observe = C.pointer(spec)
      if crop is not None:
        rec.observe_crop = C.pointer(crop)
        rec.d_observe_state = None if state is None else state.data_ptr()
      rec.d_table = obs['table'].data_ptr()
      rec.d_valid = None if obs['valid'] is None else obs['valid'].data_ptr()
      if obs['check']:
        traj.unknown.zero_()
        rec.d_unknown = traj.unknown.data_ptr()
      rec.d_view = traj.view.data_ptr()
      rec.view_stride_t = traj.view.stride()[0]
    # an empty tensor has no address; a rollout of no step reads no action
    d_actions = actions.data_ptr() if T else self._actions.data_ptr()
    if ep_rec is None:
      what = 'pcl_rollout'
      status = self._lib.pcl_rollout(self._h, d_actions, T, C.byref(self._out), C.byref(rec),
                                     self._stream())
    else:
      what = 'pcl_rollout_episodes'
      status = self._lib.pcl_rollout_episodes(self._h, d_actions, T, C.byref(self._out),
                                              C.byref(rec), C.byref(ep_rec), self._stream())
    for spec in (crop, None if att is None else att[0]):
      if spec is not None:
        _check_crop(status, what, self._h, spec)
    _lib.check(status, what, self._h)
    if obs is not None and obs['check'] and not torch.cuda.is_current_stream_capturing():
      if int(traj.unknown[0]):
        raise RuntimeError(
            'This ObservationToArray only knows array values for the characters {}, but it '
            'received an observation with a character not in that set'.format(
                ''.join(observer._value_mapping.keys())))
    return traj

  def _rollout_observer(self, observer, crop_spec):
    """What `rollout` launches for `observer`: its table (on the device, cached per
    observer object), valid mask, element type, depth, permute and whether it checks for
    unknown characters; None without an observer."""
    from pycolab_b200 import observers, rendering
    if observer is None:
      return None
    torch = _torch()
    if isinstance(observer, rendering.ObservationToFeatureArray):
      if not self.game.occlusion_in_layers or self.game.layers is not None:
        raise NotLoweredError(
            'rollout() computes feature planes from the board, so it serves games whose '
            'layers are the occluded board (occlusion_in_layers=True, no host-composed '
            'layers); call to_feature_array() after each play() for this game')
      table = observers.feature_table(observer._layers, present=self.chars)
      valid, is_3d, permute, check = None, True, observer._permute, False
    elif isinstance(observer, rendering.ObservationToArray):
      table, valid, is_3d = observer._table, observer._valid, observer._is_3d
      permute, check = observer._permute, True
    elif isinstance(observer, rendering.ObservationCharacterRepainter):
      table, valid, is_3d, permute, check = observer._table, None, False, None, False
    else:
      raise TypeError('a rollout observer is an ObservationToFeatureArray, ObservationToArray '
                      'or ObservationCharacterRepainter, not %r' % type(observer).__name__)
    depth, size = table.shape[1], table.dtype.itemsize
    windowed = crop_spec is not None
    if self._tables is None:
      self._tables = {}
    key = (id(observer), windowed)
    if key not in self._tables:
      # Over the board, pcl_rollout reads the table of each launch of <= 32 planes in turn.
      chunks = [table] if windowed else [table[:, k0:k0 + n]
                                         for k0, n in observers.plane_chunks(depth)]
      flat = np.concatenate([np.ascontiguousarray(c).reshape(-1) for c in chunks])
      t_table = torch.from_numpy(flat.view(observers._CONTAINER[size])).to(self.device)
      t_valid = None if valid is None else torch.from_numpy(valid).to(self.device)
      self._tables[key] = (observer, t_table, t_valid)    # the observer keeps its id unique
    _, t_table, t_valid = self._tables[key]

    def spec(view):
      """The pcl_observe_spec of one slot of `view` [T, B, permuted axes]."""
      base = [0, 1, 2] if is_3d else [0, 1]
      perm = list(permute) if permute is not None else base
      strides = list(view.stride())[2:]
      at = {d: strides[perm.index(d)] for d in base}
      return _lib.ObserveSpec(depth, observers._CODE_OF_SIZE[size], view.stride()[1],
                              at[0] if is_3d else 0, at[1] if is_3d else at[0],
                              at[2] if is_3d else at[1])
    return dict(table=t_table, valid=t_valid, is_3d=is_3d, permute=permute, depth=depth,
                dtype=observers.torch_dtype(table.dtype), check=check, spec=spec)

  def _host_buffers(self, slot, view_shape):
    """Pinned staging of one pipeline slot (allocated on first use)."""
    torch = _torch()
    key = (slot, tuple(view_shape))
    if self._host is None:
      self._host = {}
    if key not in self._host:
      pin = lambda shape, dt: torch.zeros(shape, dtype=dt).pin_memory()
      t = dict(actions=pin((self.batch * self.actions_per_env,), torch.int32),
               view=pin(tuple(view_shape), torch.uint8),
               reward=pin((self.batch,), torch.int32), has_reward=pin((self.batch,), torch.uint8),
               discount=pin((self.batch,), torch.float32), done=pin((self.batch,), torch.uint8))
      self._host[key] = (t, {k: v.numpy() for k, v in t.items()})
    return self._host[key]

  def play_host(self, actions, want_board=True):
    """Host-buffer step through `pcl_step_host`: int32 [B] numpy actions in,
    numpy (board [B, rows, pitch] padded, reward, has_reward, discount, done)
    views of pinned host buffers out; synchronises."""
    h, n = self._host_buffers(0, (self.batch, self.rows, self.pitch))
    n['actions'][:] = np.asarray(actions, dtype=np.int32).reshape(-1)
    _lib.check(self._lib.pcl_step_host(
        self._h, h['actions'].data_ptr(), self._actions.data_ptr(), C.byref(self._out),
        h['view'].data_ptr() if want_board else None, h['reward'].data_ptr(),
        h['has_reward'].data_ptr(), h['discount'].data_ptr(), h['done'].data_ptr(),
        self._stream()), 'pcl_step_host', self._h)
    return (n['view'][:, :, :self.cols], n['reward'], n['has_reward'], n['discount'],
            n['done'])

  def play_host_async(self, actions, slot=0, crop_spec=None, crop_state=None):
    """Pipelined host-buffer step (`pcl_step_host_async`): enqueue H2D(actions),
    the step (and, with `crop_spec`, the cropper) and the D2H of the outputs on
    the engine's copy stream, and return at once.  `host_wait(slot)` blocks until
    this call's results are valid and returns them.  With a crop spec only the
    cropped view u8 [B, rows, cols] crosses PCIe."""
    if not self._showtime:
      raise RuntimeError('play() cannot be called until its_showtime() has been called')
    if crop_spec is None:
      shape = (self.batch, self.rows, self.pitch)
    else:
      shape = (self.batch, crop_spec.rows, crop_spec.cols)
      att = self._attached
      if (att is not None and att[3] and bytes(att[0]) == bytes(crop_spec) and
          (crop_state is None or crop_state.data_ptr() == att[1].data_ptr())):
        # this very cropper runs inside the step kernel: ship its view, launch nothing more
        self._crop_dev, crop_state = att[2], att[1]
      elif self._crop_dev is None or tuple(self._crop_dev.shape) != shape:
        self._crop_dev = _torch().empty(shape, dtype=_torch().uint8, device=self.device)
    h, n = self._host_buffers(slot, shape)
    n['actions'][:] = np.asarray(actions, dtype=np.int32).reshape(-1)
    status = self._lib.pcl_step_host_async(
        self._h, h['actions'].data_ptr(), self._actions.data_ptr(), C.byref(self._out),
        None if crop_spec is None else C.addressof(crop_spec),
        None if crop_spec is None else self._crop_dev.data_ptr(),
        None if crop_state is None else crop_state.data_ptr(),
        h['view'].data_ptr(), h['reward'].data_ptr(), h['has_reward'].data_ptr(),
        h['discount'].data_ptr(), h['done'].data_ptr(), int(slot), self._stream())
    if crop_spec is not None and not self.game.float_reward:
      # a refused crop spec (a drape in the tracking list: crop() serves those) is
      # refused before the step is enqueued: no env has moved
      _check_crop(status, 'pcl_step_host_async', self._h, crop_spec)
    _lib.check(status, 'pcl_step_host_async', self._h)
    self._slot_shape[slot] = shape

  def host_wait(self, slot=0):
    """Results of the `play_host_async` call that used `slot`: numpy views of its
    pinned buffers (view, reward, has_reward, discount, done)."""
    _lib.check(self._lib.pcl_host_wait(self._h, int(slot)), 'pcl_host_wait', self._h)
    _, n = self._host_buffers(slot, self._slot_shape[slot])
    view = n['view']
    if view.shape[1:] == (self.rows, self.pitch):
      view = view[:, :, :self.cols]
    return view, n['reward'], n['has_reward'], n['discount'], n['done']

  # ------------------------------------------------------------- accessors
  def curtain(self, char):
    """Drape.curtain of every env as bool [B, rows, cols] (things.py:213-217), for the
    spec's drapes and the program's object characters alike."""
    d = (self.drape_chars + self.object_chars).index(char)
    return self._curtain_bytes(d)[:, :, :self.cols].bool()

  def _curtain_bytes(self, d):
    """Curtain of drape `d` as u8 [B, rows, pitch] (the pcl_export_curtain layout); d >=
    len(drape_chars) names object_chars[d - len(drape_chars)], which only the program's
    curtain hook serves."""
    if self.game.curtain is not None:
      out = self.game.curtain(self, d)
      if out is not None:
        return out
    out = _torch().empty((self.batch, self.rows, self.pitch), dtype=_torch().uint8,
                         device=self.device)
    _lib.check(self._lib.pcl_export_curtain(self._h, d, out.data_ptr(), self._stream()),
               'pcl_export_curtain', self._h)
    return out

  def level_rows(self, t):
    """i64 [B]: the row of each env in `t`, whose leading axis has one row for all envs,
    one per level or one per env."""
    torch = _torch()
    if t.shape[0] == self.batch:
      return torch.arange(self.batch, device=self.device)
    if t.shape[0] == 1:
      return torch.zeros(self.batch, dtype=torch.long, device=self.device)
    return self.level.long()

  def packed_bits(self, packed, rows, cols):
    """u8 [B, R, C]: cell (rows[e, i], cols[e, j]) of env e's bit rows in `packed` (i32
    [1 | n_levels | B, H, words], cell c is bit c&31 of word c>>5 as `lowering.pack_rows`
    lays it out); rows: i64 [B, R], cols: i64 [B, C]."""
    words = packed[self.level_rows(packed)[:, None, None], rows[:, :, None],
                   (cols >> 5)[:, None, :]]
    return ((words >> (cols & 31)[:, None, :].int()) & 1).to(_torch().uint8)

  def unoccluded_layers(self, chars=None):
    """Layers of `BaseUnoccludedObservationRenderer` (rendering.py:187-301) for
    every env: bool [B, len(chars), rows, cols], plane k = everywhere the owner of
    chars[k] places it, occluded or not.  Default chars: every character of the
    game, sorted (`self.chars`).  One kernel over the packed device state."""
    chars = self.chars if chars is None else ''.join(chars)
    if self.game.layers is not None:
      return self.game.layers(self, chars)
    return self._layer_planes(chars)[:, :, :, :self.cols].bool()

  def _layer_planes(self, chars):
    """The un-occluded layers of `chars` as u8 planes [B, len(chars), rows, >= cols], one
    byte per column: pcl_layers' [B, n, rows, pitch] output, or the game's layers hook."""
    torch = _torch()
    if self.game.layers is not None:
      return self.game.layers(self, chars).contiguous().view(torch.uint8)
    out = torch.empty((self.batch, len(chars), self.rows, self.pitch), dtype=torch.uint8,
                      device=self.device)
    _lib.check(self._lib.pcl_layers(self._h, chars.encode('ascii'), len(chars), out.data_ptr(),
                                    self._stream()), 'pcl_layers', self._h)
    return out

  def error_codes(self):
    torch = _torch()
    out = torch.empty((self.batch,), dtype=torch.int32, device=self.device)
    _lib.check(self._lib.pcl_error_codes(self._h, out.data_ptr(), self._stream()),
               'pcl_error_codes', self._h)
    return out

  def launch_count(self):
    n = C.c_int64()
    _lib.check(self._lib.pcl_launch_count(self._h, C.byref(n)), 'pcl_launch_count')
    return n.value

  def new_crop_state(self):
    """Corner state of one cropper object: i32 [B, 4] (row, col, initialised,
    episode), zero = not yet initialised.  One per ScrollingCropper."""
    return _torch().zeros((self.batch, 4), dtype=_torch().int32, device=self.device)

  def attach_cropper(self, crop_spec, state=None, out=None):
    """Make every later its_showtime() / play() / run() also produce this cropper's view
    of the new boards — from inside the step kernel where the game program supports it
    (`pcl_attach_cropper`: no second launch), else by a crop launch after each step.
    Returns the u8 [B, rows, cols] tensor that always holds the latest views.
    `crop_spec=None` detaches."""
    torch = _torch()
    if crop_spec is None:
      _lib.check(self._lib.pcl_attach_cropper(self._h, None, None, None), 'pcl_attach_cropper')
      self._attached = None
      return None
    if crop_spec.rows * crop_spec.cols > _lib.MAX_CROP_CELLS:
      # no entry point serves it: refuse now rather than at the first step
      _check_crop(_lib.ERR_UNSUPPORTED, 'attach_cropper', self._h, crop_spec)
    if out is None:
      out = torch.zeros((self.batch, crop_spec.rows, crop_spec.cols), dtype=torch.uint8,
                        device=self.device)
    if state is None:
      state = self.new_crop_state()
    status = self._lib.pcl_attach_cropper(self._h, C.byref(crop_spec), out.data_ptr(),
                                          state.data_ptr())
    if status == _lib.ERR_UNSUPPORTED:
      # No epilogue in this program, or a tracked drape: crop after the step.  A refused
      # spec leaves the handle's previous cropper attached; detach it, or the step kernel
      # would go on writing into that cropper's view and state after they are released.
      _lib.check(self._lib.pcl_attach_cropper(self._h, None, None, None), 'pcl_attach_cropper')
      self._attached = (crop_spec, state, out, False)
    else:
      _lib.check(status, 'pcl_attach_cropper', self._h)
      self._attached = (crop_spec, state, out, True)
    return out

  def _after_step(self):
    att = self._attached
    if att is not None and not att[3]:
      self.crop(att[0], state=att[1], out=att[2])

  def crop(self, crop_spec, state=None, out=None):
    """ScrollingCropper / FixedCropper .crop over the last boards: u8 [B, rows,
    cols].  `state` (from new_crop_state) keeps this cropper's window corners;
    None uses the single built-in slot in the plot record.  Without `out` the
    result lives in an engine-owned buffer of THIS cropper (one per `state`), valid
    until its next crop — copy to keep, as upstream (cropping.py:148-149)."""
    torch = _torch()
    shape = (self.batch, crop_spec.rows, crop_spec.cols)
    if out is None:
      # one engine-owned buffer per cropper (keyed by its corner state): two croppers
      # with the same window shape must not overwrite each other's view
      key = (shape, None if state is None else state.data_ptr())
      if self._crop_out is None:
        self._crop_out = {}
      if key not in self._crop_out:
        self._crop_out[key] = torch.empty(shape, dtype=torch.uint8, device=self.device)
      out = self._crop_out[key]
    state_ptr = None if state is None else state.data_ptr()
    curtains, ptrs = self._tracked_curtains(crop_spec)
    if ptrs is not None:
      _check_crop(self._lib.pcl_crop_tracking(self._h, C.byref(crop_spec),
                                              self._board.data_ptr(), out.data_ptr(), state_ptr,
                                              ptrs, self._stream()),
                  'pcl_crop_tracking', self._h, crop_spec)
    else:
      _check_crop(self._lib.pcl_crop(self._h, C.byref(crop_spec), self._board.data_ptr(),
                                     out.data_ptr(), state_ptr, self._stream()),
                  'pcl_crop', self._h, crop_spec)
    return out

  def _tracked_curtains(self, crop_spec):
    """(curtains, ptrs): a tracked drape's position is the median of its curtain cells, so
    the cropper kernels take the byte curtains of the drapes `crop_spec.track` names
    (cropping.py:583-596) as a MAX_TRACK array of device pointers; ptrs is None when the
    list names no drape.  Keep `curtains` alive until the launch is enqueued."""
    if not any(code < 0 for code in crop_spec.track):
      return [], None
    curtains, ptrs = [], (C.c_void_p * _lib.MAX_TRACK)()
    for i, code in enumerate(crop_spec.track):
      if code < 0:
        curtains.append(self._curtain_bytes(-code - 1))
        ptrs[i] = curtains[-1].data_ptr()
    return curtains, ptrs

  def _crop_observe(self, crop_spec, state, table, valid, is_3d, permute, unknown=None,
                    layers=None):
    """observers.crop_observe of this engine's boards through cropper `crop_spec` (its
    corner in `state`, None = the plot record's slot).  `layers`: the layer characters of
    a game built with occlusion_in_layers=False, whose un-occluded layers are cut instead
    of the board."""
    from pycolab_b200 import observers
    if crop_spec.rows * crop_spec.cols > _lib.MAX_CROP_CELLS:
      _check_crop(_lib.ERR_UNSUPPORTED, 'pcl_crop_observe', self._h, crop_spec)
    curtains, ptrs = self._tracked_curtains(crop_spec)
    planes, plane_of, pad_plane = None, None, -1
    if layers is not None:
      known = ''.join(sorted(set(ch for ch in layers if ch in self.chars)))
      plane_of = [known.find(ch) for ch in layers]
      if crop_spec.pad_char >= 0:
        pad_plane = known.find(chr(crop_spec.pad_char))
      # a source plane per character the game has (a zero plane for the others); one
      # plane stands in when there is none, read by no output plane
      planes = self._layer_planes(known or self.chars[:1])
    return observers.crop_observe(
        self._lib, self._h, crop_spec, self._board, state, ptrs, table, valid, is_3d, permute,
        self._stream(), unknown=unknown, planes=planes, plane_of=plane_of,
        pad_plane=pad_plane, check=lambda st, what: _check_crop(st, what, self._h, crop_spec))

  def pack_handoff(self, view, packed):
    """Pack `view` (u8 [B, ...], contiguous) with this step's reward / discount /
    done into `packed` u8 [>= B, PCL_HANDOFF_RECORD_BYTES] (dist.Handoff)."""
    torch = _torch()
    view_bytes = int(view[0].numel())
    assert view.dtype == torch.uint8 and view.is_contiguous() and view.shape[0] == self.batch
    assert packed.is_contiguous() and packed.shape[0] >= self.batch
    assert packed.shape[1] == ((view_bytes + 3) & ~3) + 12
    _lib.check(self._lib.pcl_pack_handoff(self._h, view.data_ptr(), view_bytes,
                                          C.byref(self._out), packed.data_ptr(),
                                          self._stream()), 'pcl_pack_handoff', self._h)
    return packed

  def pack_handoff_peers(self, view, peer_ptrs, first_row):
    """`pack_handoff` with the all-gather fused in: records go straight into row
    `first_row + env` of every rank's gather buffer (`peer_ptrs`: peer-mapped
    device pointers) over NVLink (dist.PeerHandoff)."""
    torch = _torch()
    assert view.dtype == torch.uint8 and view.is_contiguous() and view.shape[0] == self.batch
    ptrs = (C.c_void_p * len(peer_ptrs))(*[int(p) for p in peer_ptrs])
    _lib.check(self._lib.pcl_pack_handoff_peers(
        self._h, view.data_ptr(), int(view[0].numel()), C.byref(self._out), ptrs,
        len(peer_ptrs), int(first_row), self._stream()), 'pcl_pack_handoff_peers', self._h)

  def crop_handoff(self, crop_spec, crop_state, handoff_state):
    """ScrollingCropper.crop + record packing + the all-gather to every rank + the
    cross-GPU barrier as ONE kernel (`pcl_crop_handoff`, dist.FusedHandoff)."""
    _lib.check(self._lib.pcl_crop_handoff(
        self._h, C.byref(crop_spec), self._board.data_ptr(),
        None if crop_state is None else crop_state.data_ptr(), C.byref(self._out),
        C.byref(handoff_state), self._stream()), 'pcl_crop_handoff', self._h)

  # --- observation post-processors (rendering.py:304-661) over the whole batch
  def to_feature_array(self, layers, permute=None, crop_spec=None, state=None):
    """ObservationToFeatureArray: float32 one-hot planes, [B, C, rows, cols] (or
    the last three axes permuted).  A character the game lacks gives a zero plane.
    A game made with occlusion_in_layers=False copies its un-occluded layers
    (`unoccluded_layers`), as upstream copies `observation.layers`.

    With `crop_spec`, the planes of that cropper's window instead, [B, C, crop rows, crop
    cols], in one launch from the board: the window moves as `crop(crop_spec, state)`
    would move it, so call it once per step per cropper state, as `crop`.  Un-occluded
    layers are cut at the same window, off-board cells set in the pad character's plane
    (cropping.py `_do_crop`)."""
    from pycolab_b200 import observers
    torch = _torch()
    permute = observers.check_permute(permute, True, 'ObservationToFeatureArray')
    if crop_spec is not None:
      if self.game.occlusion_in_layers:
        table, lay = observers.feature_table(layers, present=self.chars), None
      else:
        table = np.zeros((128, len(layers)), dtype=np.float32)
        table[1] = 1.0                     # the cell is the layer's bit
        lay = layers
      out = self._crop_observe(crop_spec, state, table, None, True, permute, layers=lay)
      return out.view(torch.float32)
    if self.game.occlusion_in_layers:
      out = observers.observe(self._lib, self._h, self._board, self.rows, self.cols,
                              observers.feature_table(layers, present=self.chars), None,
                              True, permute, self._stream())
      return out.view(torch.float32)
    known = [k for k, ch in enumerate(layers) if ch in self.chars]
    out = torch.zeros((self.batch, len(layers), self.rows, self.cols), dtype=torch.float32,
                      device=self.device)
    if known:
      planes = self.unoccluded_layers(''.join(layers[k] for k in known))
      out[:, known] = planes.float()
    return out if permute is None else out.permute([0] + [1 + i for i in permute])

  def to_array(self, value_mapping, dtype=None, permute=None, crop_spec=None, state=None):
    """ObservationToArray: map characters to scalars ([B, rows, cols]) or vectors
    ([B, D, rows, cols]); raises RuntimeError on a character outside the mapping.
    With `crop_spec`, of that cropper's window (as `to_feature_array`); the pad
    character of a window past the board must be in the mapping too."""
    from pycolab_b200 import observers
    torch = _torch()
    table, valid, is_3d = observers.value_table(value_mapping, dtype)
    permute = observers.check_permute(permute, is_3d, 'ObservationToArray')
    unknown = torch.zeros((1,), dtype=torch.int32, device=self.device)
    if crop_spec is not None:
      out = self._crop_observe(crop_spec, state, table, valid, is_3d, permute, unknown)
    else:
      out = observers.observe(self._lib, self._h, self._board, self.rows, self.cols, table,
                              valid, is_3d, permute, self._stream(), unknown)
    if int(unknown[0]):
      raise RuntimeError(
          'This ObservationToArray only knows array values for the characters {}, but it '
          'received an observation with a character not in that set'.format(
              ''.join(value_mapping.keys())))
    return out.view(observers.torch_dtype(table.dtype))

  def repaint(self, character_mapping, crop_spec=None, state=None):
    """ObservationCharacterRepainter over every board: u8 [B, rows, cols]; with
    `crop_spec`, over that cropper's window (as `to_feature_array`)."""
    from pycolab_b200 import observers
    table = observers.repaint_table(character_mapping)
    if crop_spec is not None:
      return self._crop_observe(crop_spec, state, table, None, False, None)
    return observers.observe(self._lib, self._h, self._board, self.rows, self.cols,
                             table, None, False, None, self._stream())

  def sprite_state(self):
    """i32 [B, S, 8] device tensor of sprite records (PCL_S_* words)."""
    return self.sprites

  def frames(self):
    return self.plot[:, _lib.P_FRAME]

  def close(self):
    if getattr(self, '_h', None) is not None and self._h.value:
      self._lib.pcl_destroy(self._h)
      self._h = C.c_void_p()

  def __del__(self):
    try:
      self.close()
    except Exception:
      pass


def scrolling_crop_spec(rows, cols, sprite_index, pad_char=None, scroll_margins=(2, 3),
                        initial_offset=None, saccade=True, track=None):
  """Resolve ScrollingCropper constructor arguments (cropping.py:313-392).
  `track`: optional priority list replacing `sprite_index` — entries k > 0 mean
  sprite k - 1, k < 0 drape -k - 1 (`to_track` with several entities)."""
  if ((scroll_margins[0] is None and rows % 2 == 0) or
      (scroll_margins[1] is None and cols % 2 == 0)):
    raise ValueError("A ScrollingCropper can't perform perfectly-egocentric scrolling "
                     'with a window that has an even number of rows or columns. Either '
                     'specify looser scroll margins or use a window with odd dimensions.')
  m0 = rows // 2 if scroll_margins[0] is None else scroll_margins[0]
  m1 = cols // 2 if scroll_margins[1] is None else scroll_margins[1]
  if 2 * m0 >= rows or 2 * m1 >= cols:
    raise ValueError("A ScrollingCropper can't use scroll margins which extend to or "
                     'beyond the very centre of the scrolling window.')
  off = initial_offset if initial_offset is not None else (0, 0)
  spec = _lib.CropSpec(rows, cols, sprite_index, -1 if pad_char is None else ord(pad_char),
                       m0, m1, off[0], off[1], 1 if saccade else 0)
  if track is not None:
    if not 0 < len(track) <= _lib.MAX_TRACK or any(code == 0 for code in track):
      raise ValueError('a device cropper tracks 1..{} entities'.format(_lib.MAX_TRACK))
    for i, code in enumerate(track):
      spec.track[i] = int(code)
    spec.sprite_index = max(0, spec.track[0] - 1)
  return spec


def run_rotating(engines, actions, stream=None):
  """`len(actions)` steps from ONE C call (`pcl_run_many`): step t advances
  engines[t % len(engines)] with actions[t] (int32 device tensors).  No Python
  runs between the launches, so the call can sit inside a CUDA-graph capture."""
  torch = _torch()
  n, steps = len(engines), len(actions)
  handles = (C.c_void_p * n)(*[e._h.value for e in engines])
  outs = (C.c_void_p * n)(*[C.addressof(e._out) for e in engines])
  ptrs = (C.c_void_p * steps)()
  for t, a in enumerate(actions):
    e = engines[t % n]
    assert a.is_cuda and a.dtype == torch.int32 and a.is_contiguous()
    assert a.numel() == e.batch * e.actions_per_env
    if not e._showtime:
      raise RuntimeError('play() cannot be called until its_showtime() has been called')
    ptrs[t] = a.data_ptr()
  if stream is None:
    stream = engines[0]._stream()
  _lib.check(engines[0]._lib.pcl_run_many(handles, n, ptrs, outs, steps, stream),
             'pcl_run_many', engines[0]._h)
