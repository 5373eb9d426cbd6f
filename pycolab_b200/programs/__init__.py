"""Host side of the step programs: one module per `csrc/<program>.cu`.

Each module has `lower(engine, roles)`, which checks a set-up `Engine` against what the
kernel restates and returns its `lowering.LoweredGame`, plus the host hooks the program
needs, which `lower` stores on that game (see `LoweredGame`):
  curtain     drape curtains the device does not export: warehouse, hello, aperture, t_maze;
  layers      unoccluded layers composed on the host: t_maze;
  sync        program-private device state mirrored into the Python objects after a
              facade step: classics (the river), ordeal, t_maze, aperture, compiled;
  action_row  facade actions -> action words: fixture.
"""

from pycolab_b200.programs import (aperture, apprehend, better_scrolly, classics, compiled,
                                   fixture, hello, marauders, ordeal, scrolly_maze, shockwave,
                                   t_maze, warehouse)

# role family (the prefix of lowering.LOWERED_CLASSES' roles) -> program module
BY_FAMILY = {'scrolly': scrolly_maze, 'warehouse': warehouse, 'marauders': marauders,
             'fixture': fixture, 'classics': classics, 'better': better_scrolly,
             'aperture': aperture, 'ordeal': ordeal, 'hello': hello, 'apprehend': apprehend,
             'shockwave': shockwave, 't_maze': t_maze, 'compiled': compiled}
