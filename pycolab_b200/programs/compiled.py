"""The compiled program `csrc/compiled.cu`: MazeWalkers, plain Sprites, Scrollys, plain
drapes and a Backdrop of classes registered with `pycolab_b200.compiler`, whose update()
bodies run as device bytecode."""

import numpy as np

from pycolab_b200 import _lib
from pycolab_b200 import compiler
from pycolab_b200 import things
from pycolab_b200.errors import NotLoweredError
from pycolab_b200.lowering import (LoweredGame, _common, _plot_record, _scrolly_record,
                                   _sprite_record, _walker_meta, pack_rows, round_up)

_INT32 = (-2 ** 31, 2 ** 31 - 1)


def _register_value(owner, value):
  """An int / bool register value, or NotLoweredError."""
  if isinstance(value, (bool, np.bool_)):
    return int(bool(value)), True
  if isinstance(value, (int, np.integer)):
    if not _INT32[0] <= int(value) <= _INT32[1]:
      raise NotLoweredError('{} = {} does not fit a 32-bit register'.format(owner, value))
    return int(value), False
  raise NotLoweredError('{} holds {!r}: only int and bool values are compiled'.format(
      owner, value))


def _position_value(owner, value):
  """The (row, col) of a position attribute and its type (things.Sprite.Position or tuple),
  or NotLoweredError."""
  if ((isinstance(value, things.Sprite.Position) or type(value) is tuple) and len(value) == 2 and
      all(isinstance(x, (int, np.integer)) and not isinstance(x, (bool, np.bool_))
          for x in value)):
    words = [_register_value(owner, x)[0] for x in value]
    return words, (things.Sprite.Position if isinstance(value, things.Sprite.Position) else tuple)
  raise NotLoweredError('{} holds {!r}: a position attribute holds a Position or a tuple of '
                        'two ints'.format(owner, value))


def lower(engine, roles):
  th = engine.things
  game = LoweredGame()
  _common(engine, game, _lib.PROG_COMPILED)
  order = ''.join(game.groups)
  sprite_chars = [c for c in order if roles[c] in ('compiled.walker', 'compiled.sprite')]
  plain = [c for c in sprite_chars if roles[c] == 'compiled.sprite']
  drape_chars = [c for c in order if roles[c] in ('compiled.drape', 'compiled.scrolly')]
  if len(sprite_chars) > _lib.MAX_SPRITES or len(drape_chars) > _lib.MAX_DRAPES:
    raise NotLoweredError('too many entities for the compiled device program')
  comp = {ch: compiler.registered(type(th[ch])) for ch in order}
  # A registered Backdrop: its code runs first and writes a per-env live curtain.
  backdrop = (compiler.registered(type(engine.backdrop))
              if game.backdrop_role == 'compiled.backdrop' else None)
  compiled = [backdrop] * (backdrop is not None) + [comp[ch] for ch in order]
  if backdrop is not None:
    game.program_arg[4] = 1
    for ins in backdrop.ir:
      for x in ins[1:]:
        if isinstance(x, tuple) and x[0] == 'palette' and x[1] not in engine.backdrop.palette:
          raise NotLoweredError('{}: self.palette names {!r}, which is not a legal character of '
                                "the game's palette".format(compiler._name(backdrop.klass), x[1]))
  for ch in drape_chars:
    if type(th[ch]).curtain is not things.Drape.curtain:
      raise NotLoweredError('drape {!r} overrides `curtain`'.format(ch))
  scrollys = [ch for ch in drape_chars if roles[ch] == 'compiled.scrolly']
  # One scrolling group: its order words are the plot record's.
  groups = {th[ch]._scrolling_group for ch in sprite_chars + scrollys if ch not in plain}
  if len(groups) > 1:
    raise NotLoweredError('more than one scrolling group ({}): the compiled program keeps '
                          'one'.format(sorted(groups)))
  shapes = {th[ch].whole_pattern.shape for ch in scrollys}
  if len(shapes) > 1:
    raise NotLoweredError('Scrolly patterns of different shapes {}'.format(sorted(shapes)))
  for ch in scrollys:
    if tuple(th[ch]._board_shape) != (engine.rows, engine.cols):
      raise NotLoweredError('Scrolly {!r}: board_shape differs from the Engine board'.format(ch))
  for ch in order:                 # pattern operands must name Scrollys
    for ins in comp[ch].ir:
      if ins[0] in ('PRESCROLL', 'POSTSCROLL', 'PATTERN', 'PATANY') and isinstance(ins[1], tuple):
        if ins[1][1] in roles and roles[ins[1][1]] != 'compiled.scrolly':
          raise NotLoweredError('{}: things[{!r}] is not a Scrolly'.format(
              compiler._name(comp[ch].klass), ins[1][1]))
      if (ins[0] == 'FIELD' and isinstance(ins[1], tuple) and ins[1][1] in plain and
          ins[2] in (_lib.FIELD_VROW, _lib.FIELD_VCOL)):
        raise NotLoweredError('{}: things[{!r}].virtual_position: a plain Sprite has none'.format(
            compiler._name(comp[ch].klass), ins[1][1]))

  # the_plot keys: plot registers AUX0.. in order of first use
  keys = []
  for c in compiled:
    for key in c.keys:
      if key not in keys:
        keys.append(key)
  if len(keys) > compiler.MAX_PLOT_KEYS:
    raise NotLoweredError('the_plot keys {} need more than {} plot registers'.format(
        keys, compiler.MAX_PLOT_KEYS))
  plot_regs, plot_bools = [], []
  for key in keys:
    if key not in engine.the_plot:
      raise NotLoweredError('the_plot[{!r}] is read or written by update() but not set when '
                            'the game is lowered'.format(key))
    value, is_bool = _register_value('the_plot[{!r}]'.format(key), engine.the_plot[key])
    plot_regs.append(value)
    plot_bools.append(is_bool)

  # per-entity registers from the live objects
  registers = {}                 # char -> [(attr, is_bool)]
  values = {}
  for ch in order:
    c = comp[ch]
    ego = c.kind == 'sprite' and bool(th[ch]._egocentric_scroller)
    limit = compiler.MAX_EGOCENTRIC_REGISTERS if ego else compiler.MAX_REGISTERS[c.kind]
    if c.n_registers > limit:
      raise NotLoweredError('{} {!r} needs {} registers; {} has {}'.format(
          compiler._name(c.klass), ch, c.n_registers,
          'an egocentric walker' if ego else
          'a plain Sprite' if c.kind == 'plain' else 'a ' + c.kind, limit))
    regs = []
    values[ch] = []
    for name in c.attrs:
      if not hasattr(th[ch], name):
        raise NotLoweredError('{!r}.{} is used by update() but not set when the game is '
                              'lowered'.format(ch, name))
      owner = '{!r}.{}'.format(ch, name)
      if c.attr_types.get(name) == 'pos':
        words, kind = _position_value(owner, getattr(th[ch], name))
      else:
        value, is_bool = _register_value(owner, getattr(th[ch], name))
        words, kind = [value], (bool if is_bool else int)
      regs.append((name, kind))
      values[ch] += words
    registers[ch] = regs

  sprites = [th[c] for c in sprite_chars]
  records = []
  for s in sprites:
    v = values[s.character]
    if s.character in plain:           # registers VROW, VCOL, AUX0-AUX2
      rec = _sprite_record(s, *(v[2:] + [0, 0, 0])[:3])
      rec[_lib.S_VROW:_lib.S_VCOL + 1] = (v + [0, 0])[:2]
    elif s._egocentric_scroller:       # permits start empty (AUX0 = 0, AUX1 = never)
      rec = _sprite_record(s, 0, _lib.NEVER, (v + [0])[0])
    else:
      rec = _sprite_record(s, *(v + [0, 0, 0])[:3])
    records.append(rec)
  game.sprite_chars = ''.join(sprite_chars)
  meta = [([0, 0, 0, 0], False, False) if ch in plain else _walker_meta(th[ch], named_groups=True)
          for ch in sprite_chars]
  game.impassable = [m[0] for m in meta]
  game.confined = [m[1] for m in meta]
  game.egocentric = [m[2] for m in meta]
  game.sprites = np.array(records, dtype=np.int32).reshape(len(sprites), _lib.SPRITE_WORDS)
  for s, ch in enumerate(sprite_chars):
    if ch in plain:
      game.program_arg[3] |= 1 << s
  game.drape_chars = ''.join(drape_chars)
  game.margins = [(-1, -1)] * len(drape_chars)
  game.drape_kind = [0] * len(drape_chars)
  if shapes:
    game.pattern_rows, game.pattern_cols = shapes.pop()
    game.pattern_words = round_up((game.pattern_cols + 31) // 32 + 3, 2)
  recs = []
  for d, ch in enumerate(drape_chars):
    ent = th[ch]
    if ch in scrollys:
      rec = _scrolly_record(ent)
      rec[_lib.D_AUX0:_lib.D_AUX0 + len(values[ch])] = values[ch]
      recs.append(rec)
      game.drape_kind[d] = 1
      game.margins[d] = (-1, -1) if ent._scroll_margins is None else tuple(ent._scroll_margins)
      game.patterns[d] = pack_rows(ent.whole_pattern, game.pattern_words)
      # A pattern the code writes is per env; its curtain is kept in bits (csrc/compiled.cu).
      game.pattern_mutable[d] = any(ins[0] == 'SETPAT' for ins in comp[ch].ir)
      if game.pattern_mutable[d]:
        game.program_arg[2] |= 1 << d
        game.bits[d] = pack_rows(ent.curtain, game.bits_words)
    else:
      recs.append((values[ch] + [0] * _lib.DRAPE_WORDS)[:_lib.DRAPE_WORDS])
      game.bits[d] = pack_rows(ent.curtain, game.bits_words)
  game.drapes = np.array(recs, dtype=np.int32).reshape(len(drape_chars), _lib.DRAPE_WORDS)
  game.plot = np.array(_plot_record(**{'aux%d' % i: v for i, v in enumerate(plot_regs)}),
                       dtype=np.int32)
  game.dynamic_z = True                  # the kernel renders from the per-env z-order
  # RNG slots: the generators the code draws from, in order of first use
  streams = []
  for c in compiled:
    for stream in c.streams:
      if stream not in streams:
        streams.append(stream)
  game.rng_streams = tuple(streams)
  game.rng_from_globals = True
  game.program_arg[1] = len(streams)
  game.code = compiler.link(comp, sprite_chars, drape_chars, engine.rows, engine.cols, keys,
                            game.rng_streams, backdrop)
  game.float_reward = any(c.float_reward for c in compiled)
  game.reward_type = float if game.float_reward else int
  game.program_arg[0] = 1 if game.float_reward else 0
  game.registers = registers
  game.plot_keys = list(zip(keys, plot_bools))
  game.sync = sync
  return game


def sync(engine):
  """Registers back into the entities' attributes and the Plot's keys, each with the type its
  value had at lowering (bool stays bool, a Position stays a Position)."""
  b = engine.batched
  game = b.game
  sprites = b.sprites[0].cpu().numpy()
  drapes = b.drapes[0].cpu().numpy()
  plot = b.plot[0].cpu().numpy()
  th = engine.things
  for ch, regs in game.registers.items():
    if ch in b.sprite_chars:
      s = b.sprite_chars.index(ch)
      rec = sprites[s]
      if (game.program_arg[3] >> s) & 1:         # a plain Sprite: VROW, VCOL, AUX0-AUX2
        words = list(rec[_lib.S_VROW:_lib.S_VCOL + 1]) + list(rec[_lib.S_AUX0:])
      else:
        words = list(rec[_lib.S_AUX2 if game.egocentric[s] else _lib.S_AUX0:])
    else:
      d = b.drape_chars.index(ch)
      words = list(drapes[d][_lib.D_AUX0 if game.drape_kind[d] else 0:])
    for name, kind in regs:
      if kind in (bool, int):
        setattr(th[ch], name, kind(words.pop(0)))
      else:
        pair = (int(words.pop(0)), int(words.pop(0)))
        setattr(th[ch], name, pair if kind is tuple else kind(*pair))
  for k, (key, is_bool) in enumerate(game.plot_keys):
    word = plot[_lib.P_AUX0 + k]
    engine.the_plot[key] = bool(word) if is_bool else int(word)
  if b.backdrop_live is not None:          # the Backdrop's curtain as its code left it
    np.copyto(engine.backdrop.curtain, b.backdrop_live[0, :, :b.cols].cpu().numpy())
