#!/usr/bin/env python
"""Exercise every kernel of libpcl.so at small batch for compute-sanitizer.

    compute-sanitizer --tool memcheck  python tools/sanitize.py
    compute-sanitizer --tool racecheck python tools/sanitize.py

Small shapes (ragged last blocks, boards that are not multiples of 16 columns,
auto-resets inside the run) so that out-of-bounds accesses and shared-memory
hazards would show.  Prints one line per kernel family; the sanitizer's summary
goes to profiles/ (SURVEY.md §5).
"""

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
  import torch
  from pycolab_b200 import batched, dist as pdist, levels, lowering
  from pycolab_b200.games import (aperture, better_scrolly_maze, extraterrestrial_marauders,
                                  apprehend, fixtures, fluvial_natation, hello_world, ordeal,
                                  box_world, cued_catch, sequence_recall, shockwave, t_maze,
                                  scrolly_maze, warehouse_manager)
  from pycolab_b200.games.classics import chain_walk, cliff_walk, four_rooms
  rs = np.random.RandomState(0)

  def run(name, games, B, n_actions, steps=12, **kw):
    eng = batched.BatchedEngine(games, batch=B, **kw)
    eng.its_showtime()
    for _ in range(steps):
      a = rs.randint(0, n_actions, size=B * eng.actions_per_env).astype(np.int32)
      if eng.actions_per_env > 1:                     # fixture rows: motions + no directives
        a = a.reshape(B, eng.actions_per_env)
        a[:, -8:] = 0
        a[:, :-8] %= 9
      eng.play(torch.from_numpy(a.reshape(-1)).cuda())
    torch.cuda.synchronize()
    assert int(eng.error_codes().abs().max()) in (0, 1, 2), name
    print('ok %-28s B=%d launches=%d' % (name, B, eng.launch_count()))
    return eng

  arts = [levels.scrolly_maze_level(5 + i, world_shape=(65, 65), board_shape=(20, 37))
          for i in range(2)]
  eng = run('scrolly_maze_step', [scrolly_maze.make_game(*a) for a in arts], 7, 6)
  spec = batched.scrolling_crop_spec(9, 9, 0, pad_char=' ', scroll_margins=(None, None))
  eng.crop(spec)
  eng.crop(spec, state=eng.new_crop_state())
  # drape tracking (pcl_crop_tracking): the warp-histogram medians of both curtains, on a
  # 37-column board so the column loop takes its second pass
  drapes = batched.scrolling_crop_spec(5, 7, 0, pad_char=' ', scroll_margins=(1, 2),
                                       track=[-1, 1, -2])
  eng.crop(drapes, state=eng.new_crop_state())
  eng.crop(drapes)
  eng.unoccluded_layers()
  eng.curtain('#'), eng.curtain('@')
  eng.to_feature_array('P#@ ')
  eng.repaint({'#': '%'})
  # the window through a post-processor in one launch: drape medians, and a depth past
  # one staged chunk of the table (32 planes) in channels-last order
  eng.to_feature_array('P#@ ' * 9, permute=(1, 2, 0), crop_spec=drapes,
                       state=eng.new_crop_state())
  fused = pdist.FusedHandoff(eng, spec, eng.batch)
  fused.gather(); fused.gather()
  packed = torch.zeros((eng.batch, pdist.handoff_record_bytes(81)), dtype=torch.uint8, device='cuda')
  eng.pack_handoff(eng.crop(spec), packed)
  torch.cuda.synchronize()
  print('ok crop / layers / export / observe / handoff kernels')
  # a rollout at B=7 with quits (action 5), so envs restart inside it: the attached cropper
  # in the step kernel into its [T, B] slots, and 33 feature planes of a window per step
  from pycolab_b200 import rendering
  eng.attach_cropper(spec)
  acts = rs.randint(0, 6, size=(20, eng.batch)).astype(np.int32)
  traj = eng.rollout(torch.from_numpy(acts).cuda(), keep_attached=True,
                     observer=rendering.ObservationToFeatureArray('P#@ ' * 8 + '+'),
                     crop_spec=spec, state=eng.new_crop_state())
  eng.rollout(torch.from_numpy(acts).cuda(), observer=rendering.ObservationToFeatureArray(
      'P#@ ' * 9))                       # over the board: launches of 32 and 4 planes
  eng.attach_cropper(None)
  torch.cuda.synchronize()
  assert int(traj.done.sum()) > 0
  print('ok rollout')
  wide = levels.scrolly_maze_level(9, world_shape=(41, 161), board_shape=(12, 100))
  run('scrolly_maze_step W=100', [scrolly_maze.make_game(*wide)], 5, 5)
  # Board shapes the kernel's shared-memory layout branches on: 3 segments per row, a
  # third round of rows, the general path on a narrow board, a one-column board.
  sys.path.insert(0, os.path.join(ROOT, 'tests'))
  import scrolly_shapes as ss
  shapes = [('11x33', None, False), ('65x64', None, False), ('20x20', 80, False),
            ('9x1_nomargins', None, True)]
  for name, pitch, min_words in shapes:
    board, world, margins = ss.SHAPE[name]
    games = []
    for i in range(2):
      g = lowering.lower(ss.facade_game(*ss.open_level(40 + i, board, world), margins=margins))
      if pitch is not None:
        bd = np.zeros((g.rows, pitch), dtype=np.uint8)
        bd[:, :g.cols] = g.backdrop[:, :g.cols]
        g.backdrop, g.pitch = bd, pitch
      if min_words:
        words = ss.min_pattern_words(g.cols, g.pattern_cols)
        g.patterns = {d: lowering.pack_rows(lowering.unpack_rows(p, g.pattern_cols), words)
                      for d, p in g.patterns.items()}
        g.pattern_words = words
      games.append(g)
    run('scrolly_maze_step %s%s' % (name, '' if pitch is None else ' pitch %d' % pitch),
        games, 7, 5, steps=20)
  run('warehouse_step', [warehouse_manager.make_game(
      levels.warehouse_level(3, shape=(14, 21), num_boxes=4, num_goals=5))], 9, 6)
  run('marauders_step', [extraterrestrial_marauders.make_game(levels.marauders_level())], 6, 4,
      steps=40)
  sys.path.insert(0, os.path.join(ROOT, 'tests'))
  import golden_cases as gc
  import trajectory as tj
  run('better_scrolly_step',
      [better_scrolly_maze.make_game(tj.u8_to_art(gc.load('better_stock_L1')['art']))], 5, 6)
  for mod in (four_rooms, cliff_walk, chain_walk):
    run('classics_step ' + mod.__name__.rsplit('.', 1)[-1], [mod.make_game()], 5, 4)
  run('classics_step fluvial', [fluvial_natation.make_game()], 5, 3)
  run('aperture_step', [aperture.make_game(levels.aperture_level())], 5, 9)
  for mk in (ordeal.make_castle, ordeal.make_cavern, ordeal.make_kansas):
    g = mk()
    g.the_plot.this_chapter = mk.__name__[5:]
    run('ordeal_step ' + mk.__name__[5:], [g], 5, 5)
  # pcl_layers and pcl_export_curtain at pitch 80 > ceil16(15): the sword is a bit-row drape,
  # and the segments wholly past the board must read nothing of the rows behind the last one
  g = ordeal.make_cavern()
  g.the_plot.this_chapter = 'cavern'
  eng = run('ordeal_step cavern pitch 80', [ss.lowered(g, pitch=80)], 5, 5)
  eng.unoccluded_layers()
  eng._curtain_bytes(0)
  torch.cuda.synchronize()
  print('ok layers / export at pitch 80')
  run('hello_step', [hello_world.make_game()], 5, 6)
  run('apprehend_step (device RNG)', [apprehend.make_game()], 5, 3, steps=30)
  run('shockwave_step', [shockwave.make_game(0), shockwave.make_game(levels.shockwave_level(3, 9, 33))][:1], 5, 5, steps=40)
  run('shockwave_step 9x33', [shockwave.make_game(levels.shockwave_level(3, 9, 33))], 6, 5, steps=40)
  run('t_maze_step (device RNG)', [t_maze.make_game(1, False, 20, 2, 3, *levels.t_maze_level(s))
                                   for s in range(2)], 6, 7, steps=45)
  run('box_world_step', [box_world.make_game(g, (1, 2, 3, 4), (0, 1, 2, 3, 4), (0,), 1,
                                              random_state=np.random.RandomState(s),
                                              max_num_steps=15)
                          for g, s in ((12, 0), (12, 1), (12, 2))], 7, 6, steps=40)
  run('box_world_step 32x32', [box_world.make_game(30, (1, 2, 3, 4), (0, 1, 2, 3, 4), (0,), 1,
                                                   random_state=np.random.RandomState(4),
                                                   max_num_steps=10)], 5, 6, steps=25)
  run('cued_catch_step (device RNG)', [cued_catch.make_game(1, 2, 4, True, 0.5, 1,
                                                           art=levels.cued_catch_art(5, 14))],
      6, 3, steps=40)
  for shape in ((9, 13), (32, 64)):
    run('sequence_recall_step %dx%d' % shape,
        [sequence_recall.make_game(3, 1, 1, 0, 30, art=levels.sequence_recall_art(*shape))],
        6, 6, steps=40)
  pattern = rs.random_sample((17, 23)) < 0.2
  fx = fixtures.make_game(['           ', '   P       ', '      q    ', '           ',
                           '           ', '           '], ' ',
                          {'P': dict(impassable='#', egocentric=True, group='one'),
                           'q': dict(impassable='@', egocentric=True, group='two')},
                          {'#': dict(pattern=pattern, corner=(2, 3), margins=(2, 3), group='one'),
                           '@': dict(pattern=~pattern, corner=(1, 1), margins=None, group='two')},
                          update_schedule=[['#', '@'], ['P', 'q']], z_order='@#Pq')
  run('fixture_step (2 scrolling groups)', [fx], 5, 9)
  # Compiled scrolling games: Scrollys (one writing its pattern), egocentric walkers.
  from pycolab_b200 import compat, compiler
  compat.uninstall()
  try:
    sg = compat.load_example(os.path.join(ROOT, 'tests', 'scrolling_games.py'))
  finally:
    compat.uninstall()
  compiler.register(*sg.CLASSES)
  run('compiled_step scrolly maze', [sg.make_maze(*a) for a in arts], 7, 6, steps=20)
  run('compiled_step sampler', [sg.make_sampler(0), sg.make_sampler(1)], 5, 10, steps=30)
  print('done')


if __name__ == '__main__':
  main()
