"""Scaffolding shared by the compiled program's tests: game modules loaded through `compat`
with their classes registered, and handles that reach no device."""

import ctypes as C
import os
import sys

import numpy as np

from pycolab_b200 import _lib, compat, compiler

HERE = os.path.dirname(os.path.abspath(__file__))


def load(path):
  """Import a pycolab module through compat, leaving sys.modules as it was.  A relative
  `path` names a file under tests/."""
  saved = {k: v for k, v in sys.modules.items() if k == 'pycolab' or k.startswith('pycolab.')}
  compat.uninstall()
  try:
    return compat.load_example(os.path.join(HERE, path))
  finally:
    compat.uninstall()
    sys.modules.update(saved)


def registered(name, *extra):
  """Body of a module-scoped fixture: tests/`name` loaded, its CLASSES and the classes it
  names `extra` registered, and unregistered again at teardown."""
  mod = load(name)
  classes = list(mod.CLASSES) + [getattr(mod, k) for k in extra]
  compiler.register(*classes)
  yield mod
  compiler.unregister(*classes)


def handle(lib, spec):
  h = C.c_void_p()
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(h)) == _lib.OK
  return h


def bind(lib, h, words):
  words = np.ascontiguousarray(words, dtype=np.int32)
  return lib.pcl_bind_code(h, words.ctypes.data, len(words))
