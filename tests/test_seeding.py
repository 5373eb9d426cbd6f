"""Seeded resets (`pcl_seed_rng`, `BatchedEngine.reset(seeds=)`) without a GPU.

- The seeding rule include/pcl.h states, restated here, against NumPy's and CPython's own
  seeding.
- The ctypes mirror of PCL_SEED_* and the pcl_seed_rng signature against include/pcl.h.
- Every refusal of pcl_seed_rng on handles that reach no device (device -1, made-up
  addresses), before anything is enqueued.
- The facade's checks of `seeds`, which run before anything needs CUDA, and the choice
  between the seeding kernel and the host words in the constructor.
"""

import ctypes as C
import os
import random
import re

import numpy as np
import pytest

import boundary_sweep
import registered_games as rg
from pycolab_b200 import _lib, batched, lowering

FAKE = boundary_sweep.FAKE
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M32 = 0xffffffff
EDGE_SEEDS = (0, 1, 12345, 2 ** 31 - 1, 2 ** 31, 2 ** 32 - 1)


def _header():
  with open(os.path.join(ROOT, 'include', 'pcl.h')) as f:
    return f.read()


# ---- the rule ---------------------------------------------------------------------------

def _init_genrand(s):
  mt = [s & M32]
  for i in range(1, 624):
    mt.append((1812433253 * (mt[-1] ^ (mt[-1] >> 30)) + i) & M32)
  return mt


def _numpy_rule(s):
  return _init_genrand(s) + [624]


def _python_rule(s):
  mt = _init_genrand(19650218)
  i = 1
  for _ in range(624):
    mt[i] = ((mt[i] ^ ((mt[i - 1] ^ (mt[i - 1] >> 30)) * 1664525)) + s) & M32
    i += 1
    if i >= 624:
      mt[0], i = mt[623], 1
  for _ in range(623):
    mt[i] = ((mt[i] ^ ((mt[i - 1] ^ (mt[i - 1] >> 30)) * 1566083941)) - i) & M32
    i += 1
    if i >= 624:
      mt[0], i = mt[623], 1
  mt[0] = 0x80000000
  return mt + [624]


@pytest.mark.parametrize('seed', EDGE_SEEDS + (19650218,))
def test_the_header_rule_is_numpy_and_cpython_seeding(seed):
  assert _numpy_rule(seed) == batched._mt_state('numpy', seed).tolist()
  assert _python_rule(seed) == batched._mt_state('python', seed).tolist()
  assert _python_rule(seed) == list(random.Random(seed).getstate()[1])
  _, key, pos, _, _ = np.random.RandomState(seed).get_state()
  assert _numpy_rule(seed) == key.tolist() + [pos]


def test_ctypes_mirror_matches_the_header():
  header = _header()
  assert re.search(r'enum \{ PCL_SEED_NUMPY = 0, PCL_SEED_PYTHON = 1 \};', header)
  assert (_lib.SEED_NUMPY, _lib.SEED_PYTHON) == (0, 1)
  assert re.search(r'int pcl_seed_rng\(pcl_handle\* h, const uint8_t\* d_env_mask, '
                   r'const uint32_t\* d_seeds,\s+const int32_t\* h_kinds, int n_slots, '
                   r'void\* stream\);', header)
  restype, argtypes = _lib.SYMBOLS['pcl_seed_rng']
  assert restype is C.c_int
  assert argtypes == [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int32), C.c_int,
                      C.c_void_p]
  assert int(re.search(r'#define PCL_ABI_VERSION (\d+)', header).group(1)) == 3
  assert _lib.load().pcl_abi_version() == 3


# ---- C refusals -------------------------------------------------------------------------

def _specs():
  """{name: lowered spec} of a level of every program with generator slots, and of some
  without."""
  from pycolab_b200.games import cued_catch, sequence_recall
  from pycolab_b200.games.classics import four_rooms
  specs = dict(boundary_sweep.lowered_specs())
  specs['cued_catch'] = lowering.lower(cued_catch.make_game(1, 1, 2)).make_spec(True)
  specs['sequence_recall'] = lowering.lower(sequence_recall.make_game()).make_spec(True)
  specs['four_rooms'] = lowering.lower(four_rooms.make_game()).make_spec(True)
  for mod_name, make in (('drawn_games.py', 'make_monsters'), ('compiled_games.py', 'make_coins')):
    for mod in rg.registered(mod_name):
      specs['compiled_' + make] = lowering.lower(getattr(mod, make)(0)).make_spec(True)
  return specs


SLOTS = {'marauders': 1, 'shockwave': 1, 'apprehend': 1, 'cued_catch': 1, 'sequence_recall': 1,
         't_maze': 2, 'compiled_make_monsters': 2}


@pytest.fixture(scope='module')
def specs():
  return _specs()


def _handle(spec, state=None):
  lib = _lib.load()
  h = C.c_void_p()
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(h)) == _lib.OK
  if state is not None:
    assert lib.pcl_bind_state(h, C.byref(state)) == _lib.OK
  return lib, h


def _kinds(*kinds):
  return (C.c_int32 * max(1, len(kinds)))(*kinds)


def test_null_handle_and_null_seeds(specs):
  lib, h = _handle(specs['apprehend'], boundary_sweep._full_state())
  try:
    assert lib.pcl_seed_rng(None, None, FAKE, _kinds(1), 1, None) == _lib.ERR_INVALID
    assert lib.pcl_seed_rng(None, None, None, _kinds(1), 1, None) == _lib.ERR_INVALID
    assert lib.pcl_seed_rng(h, None, None, _kinds(1), 1, None) == _lib.ERR_INVALID
    assert lib.pcl_seed_rng(h, FAKE, None, _kinds(1), 1, None) == _lib.ERR_INVALID
  finally:
    lib.pcl_destroy(h)


def test_unbound_state_comes_before_the_program(specs):
  for name in ('apprehend', 't_maze', 'four_rooms'):
    lib, h = _handle(specs[name])
    try:
      assert lib.pcl_seed_rng(h, None, FAKE, _kinds(1, 0), SLOTS.get(name, 1), None) == \
          _lib.ERR_UNBOUND, name
    finally:
      lib.pcl_destroy(h)


def test_programs_without_generator_slots(specs):
  no_slots = [n for n in specs if n not in SLOTS]
  assert {'scrolly_maze', 'four_rooms', 'hello', 'compiled_make_coins'} <= set(no_slots)
  spec = _lib.Spec()
  spec.abi_version, spec.program = _lib.ABI_VERSION, _lib.PROG_NONE
  spec.rows, spec.cols, spec.pitch, spec.n_sprites, spec.n_drapes = 16, 16, 16, 2, 2
  for name, sp in [(n, specs[n]) for n in no_slots] + [('none', spec)]:
    lib, h = _handle(sp, boundary_sweep._full_state())
    try:
      for n in (0, 1, 2):
        # before the slot count, the kinds and d_rng are looked at
        assert lib.pcl_seed_rng(h, None, FAKE, _kinds(0, 1), n, None) == \
            _lib.ERR_UNSUPPORTED, name
        assert lib.pcl_seed_rng(h, None, FAKE, None, n, None) == _lib.ERR_UNSUPPORTED, name
    finally:
      lib.pcl_destroy(h)


def test_null_rng_words():
  # apprehend binds without generator words (the slope then comes from the template)
  from pycolab_b200.games import apprehend
  st = boundary_sweep._full_state()
  st.d_rng = None
  lib, h = _handle(lowering.lower(apprehend.make_game()).make_spec(True), st)
  try:
    assert lib.pcl_seed_rng(h, None, FAKE, _kinds(1), 1, None) == _lib.ERR_INVALID
    assert lib.pcl_seed_rng(h, FAKE, FAKE, _kinds(0), 1, None) == _lib.ERR_INVALID
  finally:
    lib.pcl_destroy(h)


@pytest.mark.parametrize('name', sorted(SLOTS))
def test_slot_count_and_kinds(specs, name):
  slots = SLOTS[name]
  lib, h = _handle(specs[name], boundary_sweep._full_state())
  try:
    for n in (-1, 0, slots - 1, slots + 1, 3, 64):
      if n != slots:
        assert lib.pcl_seed_rng(h, None, FAKE, _kinds(0, 0, 0, 0), n, None) == \
            _lib.ERR_INVALID, (name, n)
    assert lib.pcl_seed_rng(h, None, FAKE, None, slots, None) == _lib.ERR_INVALID
    for bad in (2, -1, 3, 255, 2 ** 31 - 1):
      for k in range(slots):
        kinds = [0] * slots
        kinds[k] = bad
        assert lib.pcl_seed_rng(h, None, FAKE, _kinds(*kinds), slots, None) == \
            _lib.ERR_INVALID, (name, kinds)
  finally:
    lib.pcl_destroy(h)


# ---- the facade -------------------------------------------------------------------------

def _tensor(seeds):
  """The torch tensor a parameter named 'tensor_*' stands for (tensors are made at run time)."""
  import torch
  made = {'tensor_negative': lambda: torch.tensor([0, -1, 2, 3]),
          'tensor_huge': lambda: torch.tensor([0, 1, 2 ** 32, 3]),
          'tensor_short': lambda: torch.arange(3),
          'tensor_2d': lambda: torch.zeros((4, 1), dtype=torch.int64),
          'tensor_float': lambda: torch.zeros(4),
          'tensor_bool': lambda: torch.zeros(4, dtype=torch.bool)}
  return made[seeds]() if isinstance(seeds, str) and seeds in made else seeds


def _facade_engine(batch=4, env_offset=0, draws=True):
  """A BatchedEngine shell that reaches no device: what reset()'s seed checks read."""
  import torch
  eng = batched.BatchedEngine.__new__(batched.BatchedEngine)
  eng.batch, eng.env_offset, eng.device = batch, env_offset, torch.device('cpu')
  eng.rng = torch.zeros((batch, 625), dtype=torch.int32) if draws else None
  return eng


@pytest.mark.parametrize('seeds', [-1, 2 ** 32 - 3, 2 ** 40, [0, 1, 2, -1], [0, 1, 2, 2 ** 32],
                                   np.array([0, 1, 2, -5]), np.array([0, 2 ** 32, 0, 0]),
                                   'tensor_negative', 'tensor_huge'])
def test_facade_refuses_seeds_out_of_range(seeds):
  seeds = _tensor(seeds)
  with pytest.raises(ValueError, match='2\\*\\*32'):
    _facade_engine().reset(seeds=seeds)


def test_facade_int_seed_range_counts_env_offset():
  with pytest.raises(ValueError, match='env_offset 8'):
    _facade_engine(env_offset=8).reset(seeds=2 ** 32 - 11)
  with pytest.raises(ValueError):
    _facade_engine(env_offset=8).reset(seeds=-8 - 1)
  # the last env's seed is 2**32 - 1: in range
  t = _facade_engine(env_offset=8)._seed_tensor(2 ** 32 - 12)
  assert t.tolist() == [-4, -3, -2, -1]


@pytest.mark.parametrize('seeds', [[0, 1, 2], [0, 1, 2, 3, 4], [], np.zeros((2, 2), int),
                                   'tensor_short', 'tensor_2d'])
def test_facade_refuses_the_wrong_length(seeds):
  seeds = _tensor(seeds)
  with pytest.raises(ValueError, match='4 seeds'):
    _facade_engine().reset(seeds=seeds)


@pytest.mark.parametrize('seeds', [1.5, True, np.bool_(False), 'abcd', [0, 1, 2.5, 3],
                                   [0, 1, None, 3], np.array([0.0, 1.0, 2.0, 3.0]),
                                   'tensor_float', 'tensor_bool'])
def test_facade_refuses_seeds_that_are_not_ints(seeds):
  seeds = _tensor(seeds)
  with pytest.raises(TypeError, match='ints'):
    _facade_engine().reset(seeds=seeds)


def test_facade_keeps_the_low_32_bits():
  import torch
  eng = _facade_engine()
  want = [0, 2 ** 31 - 1, -2 ** 31, -1]
  for seeds in ([0, 2 ** 31 - 1, 2 ** 31, 2 ** 32 - 1], np.array([0, 2 ** 31 - 1, 2 ** 31, 2 ** 32 - 1]),
                torch.tensor([0, 2 ** 31 - 1, 2 ** 31, 2 ** 32 - 1])):
    t = eng._seed_tensor(seeds)
    assert t.dtype == torch.int32 and t.tolist() == want
  assert eng._seed_tensor(7).tolist() == [7, 8, 9, 10]
  assert _facade_engine(env_offset=100)._seed_tensor(7).tolist() == [107, 108, 109, 110]
  assert eng._seed_tensor(np.int64(5)).tolist() == [5, 6, 7, 8]
  assert eng._seed_tensor(torch.tensor([1, 2, 3, 4], dtype=torch.uint8)).tolist() == [1, 2, 3, 4]


@pytest.mark.parametrize('seeds', [0, [0, 1, 2, 3], -1, 1.5])
def test_facade_refuses_seeds_without_generators(seeds):
  with pytest.raises(ValueError, match='draws from random generators'):
    _facade_engine(draws=False).reset(seeds=seeds)


def test_constructor_picks_the_kernel_for_32_bit_seeds():
  assert batched._device_seeded(0, 0, 4096)
  assert batched._device_seeded(2 ** 32 - 4096, 0, 4096)
  assert batched._device_seeded(2 ** 32 - 4096 - 10, 10, 4096)
  assert batched._device_seeded(np.int64(3), 5, 1)
  assert not batched._device_seeded(2 ** 32 - 4095, 0, 4096)
  assert not batched._device_seeded(-1, 0, 4)
  assert not batched._device_seeded(-4, 3, 4)        # env 0 would get -1
  assert not batched._device_seeded(0, -1, 4)
  assert not batched._device_seeded(2 ** 40, 0, 1)
  assert not batched._device_seeded(None, 0, 1)
  assert not batched._device_seeded(1.0, 0, 1)
