"""Sampled-env parity checks at full batch.  TEST INFRASTRUCTURE ONLY.

The oracle (a Python restatement of reference pycolab/engine.py:583-639 and the
example games) steps ~2x10^4 env-steps/s/core, so a 4096..16384-env batch cannot
be replayed whole.  These helpers pick a SAMPLE of env indices out of a
full-size `BatchedEngine`, step one oracle world per sampled env with that env's
own level and action stream (auto-reset = a fresh world on game-over, the
batched stand-in for "one Engine per episode", engine.py:103-104), and compare
every step's (board, reward, has_reward, discount, done) bit for bit.

Used by the batched-vs-oracle tests and by bench.py's post-timing
`parity_checked` leg (the checker, never the thing measured).
"""

import numpy as np


class Mismatch(AssertionError):
  pass


def _compare(t, env, got, want, world):
  board, reward, has, disc, done = got
  w_board, w_reward, w_disc = want
  if not np.array_equal(board, w_board):
    bad = np.argwhere(board != w_board)
    raise Mismatch('board differs at step %d env %d, first cell %s: device %r oracle %r' % (
        t, env, tuple(bad[0]), chr(board[tuple(bad[0])]), chr(w_board[tuple(bad[0])])))
  want_has = 0 if w_reward is None else 1
  if reward.dtype == np.float64:          # a game with a float reward: the float64 bits
    bits = np.float64(0.0 if w_reward is None else w_reward).view(np.int64)
    same = int(has) == want_has and np.float64(reward).view(np.int64) == bits
  else:
    same = (int(has), int(reward)) == (want_has, 0 if w_reward is None else int(w_reward))
  if not same:
    raise Mismatch('reward differs at step %d env %d: device (%d, %r) oracle %r' % (
        t, env, int(has), reward, w_reward))
  if float(disc) != float(w_disc):
    raise Mismatch('discount differs at step %d env %d: %r vs %r' % (t, env, disc, w_disc))
  if bool(done) != bool(world.game_over):
    raise Mismatch('game_over differs at step %d env %d' % (t, env))


def sprite_words(walker):
  """Words 0-4 of a sprite's device record for an oracle MazeWalker: row, col, vrow, vcol
  and the flags (bit 0 visible, bits 1-2 prior visible: 0 None, 1 False, 2 True)."""
  prior = 0 if walker.prior_visible is None else 2 if walker.prior_visible else 1
  return (walker.row, walker.col, walker.vrow, walker.vcol,
          int(bool(walker.visible)) | prior << 1)


def lockstep(engine, make_world, env_ids, actions, crop=None, curtains='', sprites='',
             pad_columns=False, on_step=None, raised=None):
  """Step `engine` (a BatchedEngine after its_showtime(), B envs) with
  actions int32 [T, B] and, for every env in `env_ids`, an oracle world built by
  make_world(env) in lockstep.  Returns the number of (env, step) pairs compared,
  resets included.  Every step compares board, reward, has_reward, discount and done;
  on request also:
    crop: (crop_spec, crop_state, make_oracle_cropper): engine.crop(crop_spec,
      state=crop_state) against a cropper that follows each oracle world.  crop_spec may
      instead be the view engine.attach_cropper() returned (crop_state unused).
    curtains: drape chars whose engine.curtain(ch) must equal the oracle drape's.
    sprites: sprite chars whose record words 0-4 must equal `sprite_words` of the
      oracle walker.
    pad_columns: the board's pitch padding stays 0.
    on_step(t, engine, worlds, outs): called after the comparison of step t (0 is
      its_showtime()), with the oracle worlds and their outputs keyed by env.
    raised: a dict, to compare the latched error words too.  Each env's word
      (engine.error_codes()) stays 0 while its oracle world raises nothing.  A world
      whose play() raises at step t must find exactly one error latched after step t:
      ENV_ERR_INDEX for an IndexError (a NumPy look-up off the board),
      ENV_ERR_EMPTY_CHOICE for a ValueError (np.random.choice of an empty list).
      lockstep then sets raised[env] = t and compares that env no further, as the
      reference's Engine would play no further.  The same holds for a world whose
      its_showtime() raises, at the first launch (t = 0) or at the launch that
      auto-resets the env."""
  import torch
  env_ids = [int(e) for e in env_ids]
  idx = torch.as_tensor(env_ids, dtype=torch.long, device=engine.device)
  T = actions.shape[0]
  def showtime(e, t):
    """A fresh world for env e at step t, and its its_showtime() output."""
    worlds[e] = make_world(e)
    if croppers is not None:
      croppers[e].set_engine(worlds[e])
    if raised is None:
      outs[e] = worlds[e].its_showtime()
      return
    try:
      outs[e] = worlds[e].its_showtime()
    except (IndexError, ValueError) as exc:
      latch(e, t, exc)

  def latch(e, t, exc):
    from pycolab_b200 import _lib
    raised[e] = t
    latched[e] = _lib.ENV_ERR_INDEX if isinstance(exc, IndexError) else _lib.ENV_ERR_EMPTY_CHOICE

  worlds, outs, latched = {}, {}, {}
  croppers = None
  if crop is not None:
    crop_spec, crop_state, make_cropper = crop
    croppers = {e: make_cropper() for e in env_ids}
  for e in env_ids:
    showtime(e, 0)
  slots = [engine.sprite_chars.index(ch) for ch in sprites]
  acts_dev = torch.from_numpy(np.ascontiguousarray(actions, dtype=np.int32)).to(engine.device)

  def pick(x):
    return x.index_select(0, idx).cpu().numpy()

  def check(t):
    if raised is not None:
      codes = pick(engine.error_codes())
      for k, e in enumerate(env_ids):
        if e in raised and raised[e] < t:
          continue
        want = latched.get(e, 0)
        if int(codes[k]) != want:
          raise Mismatch('error word at step %d env %d: device %#x oracle %#x' % (
              t, e, int(codes[k]), want))
    boards, reward, has = pick(engine.board), pick(engine.reward), pick(engine.has_reward)
    disc, done = pick(engine.discount), pick(engine.done)
    views = None
    if crop is not None:
      views = pick(crop_spec if torch.is_tensor(crop_spec) else
                   engine.crop(crop_spec, state=crop_state))
    planes = {ch: pick(engine.curtain(ch)) for ch in curtains}
    records = pick(engine.sprites) if sprites else None
    pad = pick(engine._board)[:, :, engine.cols:] if pad_columns else None
    for k, e in enumerate(env_ids):
      if raised is not None and e in raised:
        continue
      world = worlds[e]
      _compare(t, e, (boards[k], reward[k], has[k], disc[k], done[k]), outs[e], world)
      if views is not None and not np.array_equal(views[k], croppers[e].crop(outs[e][0])):
        raise Mismatch('crop differs at step %d env %d' % (t, e))
      for ch in curtains:
        if not np.array_equal(planes[ch][k], world.things[ch].curtain):
          raise Mismatch('curtain %s differs at step %d env %d' % (ch, t, e))
      for i, ch in zip(slots, sprites):
        got, want = tuple(int(x) for x in records[k, i, :5]), sprite_words(world.things[ch])
        if got != want:
          raise Mismatch('sprite %s differs at step %d env %d: device %r oracle %r' % (
              ch, t, e, got, want))
      if pad is not None and pad[k].any():
        raise Mismatch('pad columns differ from 0 at step %d env %d' % (t, e))
    if on_step is not None:
      on_step(t, engine, worlds, outs)
    return len(env_ids) - (len(raised) if raised is not None else 0)

  compared = check(0)
  for t in range(T):
    engine.play(acts_dev[t])
    for e in env_ids:
      if raised is not None and e in raised:
        continue
      if worlds[e].game_over:                 # the auto-reset rule
        showtime(e, t + 1)
      elif raised is None:
        outs[e] = worlds[e].play(int(actions[t, e]))
      else:
        try:
          outs[e] = worlds[e].play(int(actions[t, e]))
        except (IndexError, ValueError) as exc:
          latch(e, t + 1, exc)
    compared += check(t + 1)
  return compared


def replay(make_world, env, action_stream):
  """The oracle's state of one env after `action_stream` (ints, one per step the
  device took on that env) from a fresh its_showtime(), auto-reset included.
  Returns (world, last output triple)."""
  world = make_world(env)
  out = world.its_showtime()
  for a in action_stream:
    if world.game_over:
      world = make_world(env)
      out = world.its_showtime()
    else:
      out = world.play(int(a))
  return world, out


def final_state_check(engine, make_world, env_ids, action_streams, sprite_chars):
  """After the device ran `action_streams[env]` (from a fresh reset) on each
  sampled env: the last board, the last (reward, discount, done) and every
  sprite's (row, col, visible) must equal the oracle's replay."""
  import torch
  env_ids = [int(e) for e in env_ids]
  idx = torch.as_tensor(env_ids, dtype=torch.long, device=engine.device)
  boards = engine.board.index_select(0, idx).cpu().numpy()
  reward = engine.reward.index_select(0, idx).cpu().numpy()
  has = engine.has_reward.index_select(0, idx).cpu().numpy()
  disc = engine.discount.index_select(0, idx).cpu().numpy()
  done = engine.done.index_select(0, idx).cpu().numpy()
  sprites = engine.sprites.index_select(0, idx).cpu().numpy()
  steps = 0
  for k, e in enumerate(env_ids):
    world, out = replay(make_world, e, action_streams[e])
    t = len(action_streams[e])
    _compare(t, e, (boards[k], reward[k], has[k], disc[k], done[k]), out, world)
    for i, ch in enumerate(sprite_chars):
      s = world.things[ch]
      got = (int(sprites[k, i, 0]), int(sprites[k, i, 1]), bool(sprites[k, i, 4] & 1))
      want = (int(s.position[0]), int(s.position[1]), bool(s.visible))
      if got != want:
        raise Mismatch('sprite %s differs after %d steps env %d: device %r oracle %r' % (
            ch, t, e, got, want))
    steps += t
  return steps
