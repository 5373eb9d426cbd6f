"""pcl_layers and pcl_export_curtain (csrc/render.cu layers_kernel) against the oracle, over
the whole [B, n, H, pitch] output, at every case of tests/layer_cases.py.

Each case steps a BatchedEngine (auto-reset, random actions, B of 1, 5 or 37) in lock-step
with one oracle world per env.  After its_showtime() and after every step:
  * raw pcl_layers, once with every game character plus one the game lacks plus a repeat,
    once with PCL_MAX_LAYER_CHARS characters: every byte is 0 or 1, pad columns are 0, and
    [..., :W] equals oracle.engine_model.unoccluded_layers_of;
  * pcl_export_curtain of every drape at full pitch: pad columns are 0, the curtain equals
    the oracle drape's and the drape's plane of the raw pcl_layers call;
  * every output sits inside a sentinel-filled allocation whose guard bytes stay as they
    are, and every tensor the engine holds (board, records, patterns, bits, levels) is
    byte-identical before and after the calls: they read and do not write.
The programs whose curtains a host hook serves go through BatchedEngine.curtain and
unoccluded_layers in the same lock-step; pcl_layers refuses those that pcl.h names.
"""

import ctypes as C

import numpy as np
import pytest

import layer_cases as lc
from oracle import engine_model as em
from oracle import sampled_check

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5
GUARD = 4096
MAX_LAYER_CHARS = 32


def _torch():
  import torch
  return torch


class GuardedOut(object):
  """A u8 [B, n, H, pitch] output in the middle of a sentinel-filled allocation."""

  def __init__(self, shape):
    torch = _torch()
    n = int(np.prod(shape))
    self.buf = torch.full((2 * GUARD + n,), SENTINEL, dtype=torch.uint8, device='cuda')
    self.out = self.buf[GUARD:GUARD + n].view(shape)

  def guards_intact(self):
    return bool((self.buf[:GUARD] == SENTINEL).all()) and bool((self.buf[-GUARD:] == SENTINEL).all())


def _held(eng):
  """Every tensor the engine holds, in attributes, dicts and lists."""
  torch = _torch()
  for k, v in sorted(vars(eng).items()):
    vals = v.items() if isinstance(v, dict) else enumerate(v) if isinstance(v, list) else [(k, v)]
    for kk, t in vals:
      if torch.is_tensor(t) and t.numel():
        yield '%s[%s]' % (k, kk), t


def _stream():
  return C.c_void_p(_torch().cuda.current_stream().cuda_stream)


def _layers(eng, chars):
  from pycolab_b200 import _lib
  g = GuardedOut((eng.batch, len(chars), eng.rows, eng.pitch))
  _lib.check(eng._lib.pcl_layers(eng._h, chars.encode('ascii'), len(chars), g.out.data_ptr(),
                                 _stream()), 'pcl_layers', eng._h)
  return g


def _export(eng, d):
  from pycolab_b200 import _lib
  g = GuardedOut((eng.batch, eng.rows, eng.pitch))
  _lib.check(eng._lib.pcl_export_curtain(eng._h, d, g.out.data_ptr(), _stream()),
             'pcl_export_curtain', eng._h)
  return g


def _char_lists(eng):
  """Every game character, one it lacks and a repeat; and a PCL_MAX_LAYER_CHARS list."""
  absent = [chr(c) for c in range(33, 127) if chr(c) not in eng.chars]
  first = eng.chars + absent[0] + eng.chars[0]
  full = list(eng.chars + eng.chars[-1]) + absent[1:MAX_LAYER_CHARS - len(eng.chars)]
  np.random.RandomState(len(eng.chars)).shuffle(full)
  assert len(full) == MAX_LAYER_CHARS
  return [first, ''.join(full)]


def _first_pad_byte(a, W):
  bad = np.argwhere(a[..., W:] != 0)
  return None if not len(bad) else tuple(bad[0][:-1]) + (W + bad[0][-1],)


def _check_frame(t, eng, worlds):
  torch = _torch()
  W = eng.cols
  before = [(name, x.clone()) for name, x in _held(eng)]
  raw = [(chars, _layers(eng, chars)) for chars in _char_lists(eng)]
  curtains = [_export(eng, d) for d in range(len(eng.drape_chars))]
  torch.cuda.synchronize()
  changed = [name for (name, x), (_, y) in zip(before, _held(eng)) if not torch.equal(x, y)]
  assert not changed, 't=%d: the layers calls wrote %s' % (t, changed)
  for what, g in [(c, g) for c, g in raw] + [('curtain %d' % d, g) for d, g in enumerate(curtains)]:
    assert g.guards_intact(), 't=%d %s: a guard byte changed' % (t, what)
  for chars, g in raw:
    planes = g.out.cpu().numpy()
    assert planes.max() <= 1, 't=%d %r: a byte other than 0 or 1' % (t, chars)
    pad = _first_pad_byte(planes, W)
    assert pad is None, 't=%d %r: pad byte %s = %d' % (t, chars, pad, planes[pad])
    for e, w in worlds.items():
      want = em.unoccluded_layers_of(w.backdrop, w.things, sorted(set(chars) | set(w.things)))
      for k, ch in enumerate(chars):
        np.testing.assert_array_equal(planes[e, k, :, :W], want[ch],
                                      err_msg='t=%d env %d plane %d %r' % (t, e, k, ch))
  planes = raw[0][1].out
  for d, g in enumerate(curtains):
    ch = eng.drape_chars[d]
    got = g.out.cpu().numpy()
    pad = _first_pad_byte(got, W)
    assert pad is None, 't=%d curtain %r: pad byte %s = %d' % (t, ch, pad, got[pad])
    assert torch.equal(g.out, planes[:, raw[0][0].index(ch)]), 't=%d curtain %r' % (t, ch)
    for e, w in worlds.items():
      np.testing.assert_array_equal(got[e, :, :W], w.things[ch].curtain,
                                    err_msg='t=%d env %d curtain %r' % (t, e, ch))


def _engine(built, binding, B):
  from pycolab_b200 import batched
  return batched.BatchedEngine(list(built.games), batch=B, rng_seed=built.rng_seed,
                               share_levels=binding != lc.PER_ENV)


class Restarts(object):
  """on_step for sampled_check.lockstep: counts the envs an oracle world was rebuilt for
  (restarts), and the compared frames in which the device's '@' record holds a live stale
  coin slot (AUX0 >= 0: a coin collected on a step without '@' motion)."""

  def __init__(self, then=None):
    self.then, self.worlds, self.restarts, self.stale = then, {}, 0, 0

  def __call__(self, t, eng, worlds, outs):
    from pycolab_b200 import _lib
    self.restarts += sum(e in self.worlds and w is not self.worlds[e] for e, w in worlds.items())
    self.worlds = dict(worlds)
    if '@' in eng.drape_chars and eng.game.program == _lib.PROG_SCROLLY_MAZE:
      coins = eng.drapes[:, eng.drape_chars.index('@'), _lib.D_AUX0]
      self.stale += int((coins >= 0).sum())
    if self.then is not None:
      self.then(t, eng, worlds, outs)


@pytest.mark.parametrize('case', lc.CASES, ids=[c.id for c in lc.CASES])
def test_layers_and_curtains_vs_oracle(case):
  """One case of layer_cases: every frame through _check_frame.  Envs restart inside the
  run, and a scrolly_maze case of more than one env shows the coin window's stale slot."""
  B, built = case.batch, case.build()
  assert all(g.pitch == case.pitch for g in built.games)
  eng = _engine(built, case.binding, B)
  eng.its_showtime()
  actions = built.draw(np.random.RandomState(B + case.pitch), built.steps, B)
  seen = Restarts(lambda t, eng, worlds, outs: _check_frame(t, eng, worlds))
  sampled_check.lockstep(eng, built.make_world, range(B), actions, pad_columns=True,
                         on_step=seen)
  assert seen.restarts > 0
  if case.program == 'scrolly_maze' and B > 1:
    assert seen.stale > 0


@pytest.mark.parametrize('program,hook,build', lc.HOOK_CASES, ids=[c[0] for c in lc.HOOK_CASES])
def test_host_hooks_vs_oracle(program, hook, build):
  """BatchedEngine.curtain for every drape (and object character) and, where the facade
  serves them, unoccluded_layers; pcl_layers refuses the programs pcl.h names."""
  from pycolab_b200 import _lib
  built = build()
  B = 5
  eng = _engine(built, lc.POOL if len(built.games) > 1 else lc.SHARED, B)
  eng.its_showtime()
  if hook == 'curtain':
    out = GuardedOut((B, 1, eng.rows, eng.pitch))
    got = eng._lib.pcl_layers(eng._h, eng.chars[:1].encode('ascii'), 1, out.out.data_ptr(),
                              _stream())
    assert got == _lib.ERR_UNSUPPORTED
    assert out.guards_intact() and bool((out.out == SENTINEL).all())

  def check(t, eng, worlds, outs):
    for ch in eng.drape_chars + eng.object_chars:
      got = eng.curtain(ch).cpu().numpy()
      for e, w in worlds.items():          # a level without the object: an empty curtain
        want = w.things[ch].curtain if ch in w.things else np.zeros_like(got[e])
        np.testing.assert_array_equal(got[e], want, err_msg='t=%d env %d %r' % (t, e, ch))
    if hook == 'layers':
      planes = eng.unoccluded_layers().cpu().numpy()
      for e, w in worlds.items():
        want = em.unoccluded_layers_of(w.backdrop, w.things, eng.chars)
        for k, ch in enumerate(eng.chars):
          np.testing.assert_array_equal(planes[e, k], want[ch],
                                        err_msg='t=%d env %d %r' % (t, e, ch))
  actions = built.draw(np.random.RandomState(3), built.steps, B)
  seen = Restarts(check)
  sampled_check.lockstep(eng, built.make_world, range(B), actions, on_step=seen)
  assert seen.restarts > 0


def test_scrolly_maze_facade_layers_through_a_pick_up():
  """Engine(occlusion_in_layers=False) on scrolly_maze: Observation.layers == the oracle's
  at every frame.  The walk quits whenever the player stands on a coin the '@' drape has
  not yet collected (layer_cases.coin_under_player, after a scroll onto it): that quit
  collects the coin with no '@' motion, so the frame after it shows the coin window's
  stale slot.  Episodes run until three such frames have been compared, each with the '@'
  record's AUX0 >= 0 on the device and the collected cell still in the oracle's curtain."""
  import scrolly_shapes as ss
  from pycolab_b200 import _lib
  art = ss.shape_level('20x20', 3)
  rs = np.random.RandomState(5)
  stale = 0
  for episode in range(30):
    game = ss.facade_game(*art, occlusion_in_layers=False)
    world = ss.oracle_world(*art)
    obs, _, _ = game.its_showtime()
    world.its_showtime()
    for t in range(200):
      want = em.unoccluded_layers_of(world.backdrop, world.things, sorted(obs.layers))
      for ch, layer in obs.layers.items():
        np.testing.assert_array_equal(layer, want[ch], err_msg='episode %d t=%d %r' % (
            episode, t, ch))
      if game.game_over:
        break
      pending = lc.coin_under_player(world)
      a = 5 if pending else int(rs.choice(5))
      obs, reward, _ = game.play(a)
      out = world.play(a)
      assert reward == out[1]
      if pending:
        coins = world.things['@']
        r, c = coins.corner
        window = coins.pattern[r:r + world.rows, c:c + world.cols]
        assert (coins.curtain & ~window).sum() == 1 and reward == 100
        rec = game._batched.drapes[0, game._batched.drape_chars.index('@')].cpu().numpy()
        assert rec[_lib.D_AUX0] >= 0, rec
        stale += 1
    if stale >= 3:
      break
  assert stale >= 3
