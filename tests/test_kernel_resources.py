"""CPU test of what ptxas made of the scrolly_maze step kernel in the built libpcl.so.

A 4096-env launch runs in one wave on an H100 only while 8 four-warp blocks fit on an
SM: at most 64 registers per thread, and no local-memory stack (spills).  The shared
memory side of that budget is a static_assert in scrolly_maze.cu.
"""

import os
import re
import shutil
import subprocess

import pytest

from pycolab_b200 import _lib


def _cuobjdump():
  for cand in (shutil.which('cuobjdump'),
               os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'cuobjdump')):
    if cand and os.access(cand, os.X_OK):
      return cand
  return None


def _resource_usage(lib):
  """{mangled kernel name: {'REG': n, 'STACK': n, ...}} from cuobjdump."""
  out = subprocess.run([_cuobjdump(), '--dump-resource-usage', lib], check=True,
                       capture_output=True, text=True).stdout
  usage, name = {}, None
  for line in out.splitlines():
    m = re.match(r'\s*Function (\S+):', line)
    if m:
      name = m.group(1)
    elif name and 'REG:' in line:
      usage[name] = {k: int(v) for k, v in re.findall(r'(\w+):(\d+)', line)}
      name = None
  return usage


@pytest.mark.skipif(_cuobjdump() is None, reason='cuobjdump not found')
def test_scrolly_maze_step_fits_eight_blocks_per_sm():
  assert os.path.exists(_lib.LIB_PATH), 'build libpcl.so first'
  kernels = {n: u for n, u in _resource_usage(_lib.LIB_PATH).items() if 'scrolly_maze_step' in n}
  assert kernels, 'no scrolly_maze_step in %s' % _lib.LIB_PATH
  for name, u in kernels.items():
    assert u['REG'] <= 64, (name, u)
    assert u['STACK'] == 0, (name, u)
