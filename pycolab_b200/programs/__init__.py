"""Host side of the step programs: one module per `csrc/<program>.cu`.

Each module has `lower(engine, roles)`, which checks a set-up `Engine` against what the
kernel restates and returns its `lowering.LoweredGame`, plus the host hooks the program
needs, which `lower` stores on that game (see `LoweredGame`):
  curtain     drape curtains the device does not export: warehouse, hello, aperture, t_maze,
              box_world (its object grid);
  layers      unoccluded layers composed on the host: t_maze, box_world;
  sync        program-private device state mirrored into the Python objects after a
              facade step: classics (the river), ordeal, t_maze, aperture, compiled, box_world,
              cued_catch, sequence_recall;
  python_reward  the Python type of each step's reward where it varies: cued_catch;
  action_row  facade actions -> action words: fixture.
"""

from pycolab_b200.programs import (aperture, apprehend, better_scrolly, box_world, classics,
                                   compiled, cued_catch, fixture, hello, marauders, ordeal,
                                   scrolly_maze, sequence_recall, shockwave, t_maze, warehouse)

# role family (the prefix of lowering.LOWERED_CLASSES' roles) -> program module
BY_FAMILY = {'scrolly': scrolly_maze, 'warehouse': warehouse, 'marauders': marauders,
             'fixture': fixture, 'classics': classics, 'better': better_scrolly,
             'aperture': aperture, 'ordeal': ordeal, 'hello': hello, 'apprehend': apprehend,
             'shockwave': shockwave, 't_maze': t_maze, 'compiled': compiled,
             'box_world': box_world, 'cued_catch': cued_catch,
             'sequence_recall': sequence_recall}
