"""oracle/sampled_check.lockstep under an episode time limit (BatchedEngine.set_time_limit).

Upstream pycolab has no time limit, so the oracle worlds have none either.  `TimeLimited`
adds the rule to one world from the outside, as a user wraps an Engine: after its L-th
play() a world the game has not ended reports game_over 2 (DONE_TIME_LIMIT), which
lockstep's auto-reset rule then rebuilds like any ended world.  `lockstep` runs
sampled_check.lockstep over such worlds and also compares every step's done value itself,
where sampled_check compares only whether the episode is over.
"""

import numpy as np

from oracle import sampled_check as sc


class TimeLimited(object):
  """An oracle world whose episode also ends at its L-th play(): game_over is 0 running,
  1 ended by the game, 2 ended by the limit.  Everything else is the world's."""

  def __init__(self, world, limit):
    self._world, self._limit = world, limit
    self._plays, self._cut = 0, False

  def its_showtime(self):
    return self._world.its_showtime()

  def play(self, action):
    out = self._world.play(action)
    self._plays += 1
    self._cut = 0 < self._limit <= self._plays and not self._world.game_over
    return out

  @property
  def game_over(self):
    return 1 if self._world.game_over else 2 if self._cut else 0

  def __getattr__(self, name):
    return getattr(self._world, name)


def lockstep(engine, make_world, env_ids, actions, time_limit, on_step=None, **kw):
  """sampled_check.lockstep with every world wrapped in TimeLimited(world, time_limit), and
  the exact done value of every compared env checked after every step.  Returns
  (pairs compared, how many (env, step) pairs the limit ended)."""
  import torch
  env_ids = [int(e) for e in env_ids]
  idx = torch.as_tensor(env_ids, dtype=torch.long, device=engine.device)
  raised = kw.get('raised')
  cut = [0]

  def check_done(t, eng, worlds, outs):
    done = eng.done.index_select(0, idx).cpu().numpy()
    for k, e in enumerate(env_ids):
      if raised is not None and e in raised:
        continue
      want = worlds[e].game_over
      if int(done[k]) != want:
        raise sc.Mismatch('done differs at step %d env %d: device %d oracle %d' % (
            t, e, int(done[k]), want))
    cut[0] += int(np.count_nonzero(done == 2))
    if on_step is not None:
      on_step(t, eng, worlds, outs)

  compared = sc.lockstep(engine, lambda e: TimeLimited(make_world(e), time_limit), env_ids,
                         actions, on_step=check_done, **kw)
  return compared, cut[0]
