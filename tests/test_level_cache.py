"""The level cache (include/crafter_b200.h, cr_set_level_cache / cr_fill_level_cache) on the product's kernels on the
SIMT emulator (tests/simt/simt_level_cache.cpp).

* A run with the cache equals the same run without it after every call -- reward, done, the obs of every kind of
  step, the terminal outputs and every state buffer, final_world_seed included -- for a batch that mixes level -1,
  fixed levels and sampled envs across many auto-resets, at the default geometry and at an odd one.
* Filled rows equal the C oracle's fresh worlds (tests/oracle_levels.py): terrain, creatures in slot order, n.
* A row is used only when its tag matches: corrupted tags and seeds rewritten after the fill still play exactly,
  a refill regenerates only the mismatched rows, and a matched row (poisoned on purpose) is what gets installed.
* A world that overflows a small slot arena raises the same error bit from the cache as generated.
* ptxas: no spills in the kernels the cache added or changed."""
import ctypes

import numpy as np
import pytest

from crafter_b200 import _cabi
from crafter_b200 import state as state_lib
from crafter_b200 import vector
from tests import hostsim_env
from tests import oracle_levels
from tests.test_build_properties import ptxas  # noqa: F401  (fixture)
from tests.test_level_sampler import SAMPLED, SimtSamplerEnv, simt_sampler_lib
from tests.test_levels import KINDS

NM_WORLD_SEED, NM_EPISODE = 1, 2
ERR_SLOT_OVERFLOW = 1
_LIB = []


def simt_cache_lib():
  """tests/simt/simt_level_cache.cpp: the sampler build plus hs_set_level_cache and hs_fill_level_cache."""
  if not _LIB:
    here = hostsim_env.HERE
    src = here / 'simt' / 'simt_level_cache.cpp'
    out = here / 'simt' / '_build' / 'libsimt_level_cache.so'
    deps = [src] + [here / 'simt' / n for n in ('simt_level_sampler.cpp', 'simt_levels.cpp', 'simt_symbolic.cpp',
                                                 'simt_local.cpp', 'simt_env.cpp', 'simt.h')] + list(
        (here.parent / 'crafter_b200' / 'csrc').glob('*.h')) + [here.parent / 'include' / 'crafter_b200.h']
    hostsim_env._compile(out, src, deps)
    L = ctypes.CDLL(str(out))
    base = simt_sampler_lib()
    for name in ('hs_create', 'hs_destroy', 'hs_reset', 'hs_step', 'hs_render', 'hs_semantic', 'hs_step_local',
                 'hs_local', 'hs_set_final_local', 'hs_step_symbolic', 'hs_symbolic', 'hs_set_final_symbolic',
                 'hs_set_level_buffers', 'hs_set_levels', 'hs_set_level_table', 'hs_sample_levels', 'hs_seed_only'):
      getattr(L, name).argtypes = getattr(base, name).argtypes
    L.hs_last_error.restype = ctypes.c_char_p
    L.hs_simt_blocks.restype = ctypes.c_long
    L.hs_set_level_cache.argtypes = [ctypes.c_void_p] * 6 + [ctypes.c_int]
    L.hs_fill_level_cache.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
    _LIB.append(L)
  return _LIB[0]


class SimtCacheEnv(SimtSamplerEnv):
  """SimtSamplerEnv with a level cache in caller-owned numpy buffers, as a cr_set_level_cache caller holds it."""

  @staticmethod
  def _load(max_obj_tiles):
    assert max_obj_tiles is None
    return simt_cache_lib()

  def set_level_cache(self, rows=None):
    rows = rows or self.t_cap
    self.c_mat = np.zeros((rows, self.area[0] * self.area[1]), np.uint8)
    self.c_ents = np.zeros((rows, self.capacity), np.int64)
    self.c_meta = np.zeros((rows, 2), np.int32)
    self.c_tag = np.full(rows, -1, np.int32)
    self.c_row = np.full((self.B, 2), -1, np.int32)
    self._check(self._L.hs_set_level_cache(self.h, *(a.ctypes.data for a in (
        self.c_mat, self.c_ents, self.c_meta, self.c_tag, self.c_row)), rows))

  def remove_level_cache(self):
    self._check(self._L.hs_set_level_cache(self.h, None, None, None, None, None, 0))

  def fill(self, first=0, count=None):
    self._check(self._L.hs_fill_level_cache(self.h, first, int(self.t_n[0]) if count is None else count))

  def cached_rows(self):
    """The host restatement of wg_cached_row for every env: the row its prefetched world is copied from, or -1."""
    nm = self.state['next_meta']
    row = self.c_row[np.arange(self.B), nm[:, NM_EPISODE] & 1]
    ok = (row >= 0) & (row < len(self.c_tag))
    hit = ok & (self.c_tag[np.where(ok, row, 0)] == nm[:, NM_WORLD_SEED])
    return np.where(hit, row, -1)


class Pair:
  """The same batch twice, `plain` without and `cached` with a level cache; every call goes to both and the two are
  compared after it: the call's outputs, every state buffer and the terminal outputs."""

  def __init__(self, K, seed, length, **kwargs):
    make = lambda: SimtCacheEnv(num_envs=K, seed=seed, length=length, auto_reset=True, **kwargs)
    self.plain, self.cached = make(), make()
    self.hits = 0  # worlds the cached env copied from the cache

  def both(self, fn):
    return fn(self.plain), fn(self.cached)

  def check(self, where):
    a, b = self.plain, self.cached
    for k, v in a.state.items():
      assert (v == b.state[k]).all(), (where, k, np.flatnonzero((v != b.state[k]).reshape(len(v), -1).any(1)))
    for name in ('final_world_seed', 'level', 'final_semantic', 'final_local', 'final_symbolic', 'final_obs', 'obs'):
      x, y = getattr(a, name), getattr(b, name)
      assert (x is None) == (y is None) and (x is None or (x == y).all()), (where, name)

  def reset(self, mask=None, kind='rgb'):
    self.hits += int((self.cached.cached_rows() >= 0).sum())  # what this reset installs (prefetched worlds)
    oa, ob = self.both(lambda e: e.reset(mask, kind=kind).copy())
    assert (oa == ob).all()
    self.check('reset')

  def step(self, t, actions, kind):
    ra, rb = self.both(lambda e: [x.copy() for x in e.step(actions, kind)])
    for x, y, what in zip(ra, rb, ('obs', 'reward', 'done')):
      assert (x == y).all(), (t, kind, what)
    self.check((t, kind))
    # the envs that finished had their next world built in this step, from the cache where it holds the world
    self.hits += int(((self.cached.cached_rows() >= 0) & rb[2].astype(bool)).sum())
    return rb[2].astype(bool)


def mixed_batch(pair, K, table, weights):
  """Envs 0 mod 3 on level -1, 1 mod 3 fixed, the rest sampled, the table registered, the cache filled."""
  levels = np.where(np.arange(K) % 3 == 1, 1000 + np.arange(K), -1).astype(np.int32)
  pair.both(lambda e: e.set_level_table(table, weights, cap=len(table) + 3))
  pair.cached.set_level_cache()
  pair.cached.fill()
  pair.both(lambda e: e.set_levels(levels, np.arange(K) % 3 == 1))
  pair.both(lambda e: e.sample_levels(np.arange(K) % 3 == 2))


@pytest.mark.parametrize('geometry', [dict(), dict(area=(37, 29), view=(7, 9), size=(35, 45))],
                         ids=['default', 'odd_area'])
def test_a_cached_run_equals_the_run_without_the_cache(geometry):
  K, seed, length = 13, 61, 4
  pair = Pair(K, seed, length, **geometry)
  table = np.array([5, 1234567, 2 ** 31 - 2, 0, 99, 31337], np.int64)
  mixed_batch(pair, K, table, [3, 1, 2, 0, 2, 1])
  pair.reset()
  sampled = np.arange(K) % 3 == 2
  rs = np.random.RandomState(seed)
  episodes = 0
  for t in range(20):
    actions = rs.randint(0, 17, K).astype(np.int32)
    done = pair.step(t, actions, KINDS[t % 3])
    episodes += int(done.sum())
    rows = pair.cached.cached_rows()
    assert (rows[~sampled] == -1).all(), 'an env on level -1 or a fixed level was served from the cache'
    assert (rows[sampled] >= 0).all(), 'a sampled world of a filled table was not found in the cache'
  assert episodes >= 3 * K and pair.hits >= K, (episodes, pair.hits)
  assert {int(v) for v in pair.cached.final_world_seed[sampled]} <= set(table.tolist())


def test_rows_equal_the_oracle_worlds():
  area = (64, 64)
  env = SimtCacheEnv(num_envs=2, seed=3)
  seeds = np.array([0, 77, 2 ** 31 - 2, 424242, 9], np.int64)
  env.set_level_table(seeds)
  env.set_level_cache()
  env.fill()
  geometry = oracle_levels._key(dict(area=area))
  ents = env.c_ents.view(state_lib.ENT_DTYPE)
  for i, s in enumerate(seeds):
    want = oracle_levels.fresh_world(int(s), geometry)
    assert env.c_tag[i] == s
    assert (env.c_mat[i].reshape(area) == want['mat']).all(), (i, 'terrain')
    creatures = want['objs'][1:]  # slot 1 is the player
    n, valid = env.c_meta[i]
    assert n == 2 + len(creatures) and valid == 1, (i, n, valid)
    got = np.array([[e['type'], e['x'], e['y'], e['health'], e['aux'] if e['type'] != 2 else 0, 0]
                    for e in ents[i, 2:n]], np.int64).reshape(-1, 6)
    assert (got == creatures).all(), (i, 'creatures')


def test_mismatched_tags_fall_back_and_a_refill_regenerates_only_them():
  K, seed, length = 7, 5, 3
  pair = Pair(K, seed, length)
  table = np.array([10, 20, 30, 40], np.int64)
  pair.both(lambda e: e.set_level_table(table))
  c = pair.cached
  c.set_level_cache()
  c.fill()
  pair.both(lambda e: e.sample_levels())
  pair.reset()
  rs = np.random.RandomState(1)
  for t in range(18):
    if t == 3:
      c.c_tag[1] = 999  # corrupted: row 1 no longer claims seed 20
    if t == 6:
      pair.both(lambda e: e.t_seeds.__setitem__(2, 555))  # the caller rewrote a seed after the fill
    if t == 9:
      c.c_tag[0] = -1
    pair.step(t, rs.randint(0, 17, K).astype(np.int32), KINDS[t % 3])
  # a refill regenerates rows 0, 1 (tags off) and 2 (seed changed); row 3 matches and is left as it is
  c.c_mat[3] = 0xEE
  c.fill()
  assert c.c_tag.tolist() == [10, 20, 555, 40] and (c.c_mat[3] == 0xEE).all()
  fresh = SimtCacheEnv(num_envs=1, seed=0)
  fresh.set_level_table([10, 20, 555])
  fresh.set_level_cache()
  fresh.fill()
  for i in range(3):
    assert (c.c_mat[i] == fresh.c_mat[i]).all() and (c.c_meta[i] == fresh.c_meta[i]).all(), i
    n = c.c_meta[i][0]
    assert (c.c_ents[i, 2:n] == fresh.c_ents[i, 2:n]).all(), i
  # the poisoned row is matched, so it is what a sampled env that draws seed 40 installs
  one = SimtCacheEnv(num_envs=2, seed=0, auto_reset=True, length=3)
  one.set_level_table([40])
  one.set_level_cache()
  one.c_mat[:], one.c_ents[:], one.c_meta[:], one.c_tag[:] = c.c_mat[3], c.c_ents[3], c.c_meta[3], 40
  one.sample_levels()
  one.reset()
  assert (one.state['mat'] == 0xEE).all(), 'the matched row was not copied in'


def test_a_slot_overflow_from_the_cache_raises_the_same_error():
  K, seed = 4, 17
  pair = Pair(K, seed, 3, slot_capacity=8)
  table = np.array([3, 4, 5], np.int64)
  pair.both(lambda e: e.set_level_table(table))
  pair.cached.set_level_cache()
  pair.cached.fill()
  assert (pair.cached.c_meta[:, 1] == 3).any(), 'no world of the table overflows 8 slots'
  pair.both(lambda e: e.sample_levels())
  pair.reset()
  for t in range(6):
    pair.step(t, np.zeros(K, np.int32), 'semantic')
  errors = pair.cached.errors()
  assert (errors & ERR_SLOT_OVERFLOW).any() and (errors == pair.plain.errors()).all()


def test_fill_touches_no_env_state_and_needs_a_table_and_a_cache():
  env = SimtCacheEnv(num_envs=3, seed=8, auto_reset=True, length=3)
  with pytest.raises(RuntimeError, match='no level table'):
    env.fill(0, 1)
  env.set_level_table([7, 8, 9])
  with pytest.raises(RuntimeError, match='no level cache'):
    env.fill(0, 3)
  with pytest.raises(RuntimeError, match='mat without'):
    env._check(env._L.hs_set_level_cache(env.h, env.level.ctypes.data, None, None, None, None, 2))
  env.sample_levels()
  env.reset()
  before = {k: v.copy() for k, v in env.state.items()}
  env.set_level_cache(rows=2)  # fewer rows than entries: entry 2 is not cached
  env.fill(0, 3)
  assert all((v == before[k]).all() for k, v in env.state.items())
  assert env.c_tag.tolist() == [7, 8]
  env.fill(1, 5)  # nothing left to do
  env.remove_level_cache()
  env.step(np.zeros(3, np.int32))  # no cache registered: generated as before


def test_vector_env_passes_the_cache_through():
  calls = []

  class FakeEnv:

    def set_level_cache(self, enabled=True):
      calls.append(enabled)

  venv = vector.VectorEnv.__new__(vector.VectorEnv)
  venv.env = FakeEnv()
  venv.set_level_cache()
  venv.set_level_cache(False)
  assert calls == [True, False]


def test_abi_is_extended_not_changed():
  names = [f[0] for f in _cabi.CrState._fields_]
  assert len(names) == 24 and _cabi.ABI_VERSION == 6
  assert {'cr_set_level_cache', 'cr_fill_level_cache'} <= set(_cabi.EXPORTS)
  header = (hostsim_env.HERE.parent / 'include' / 'crafter_b200.h').read_text()
  assert 'int cr_set_level_cache(' in header and 'int cr_fill_level_cache(' in header


def test_cache_kernels_do_not_spill(ptxas):  # noqa: F811
  for kernel in ('k_seed', 'k_fill_seed', 'k_fill_tag', 'k_wg_mat', 'k_wg_obj'):
    found = {targs: v for (name, targs), v in ptxas.items() if name == kernel}
    assert found and all(v.get('spill', 0) == 0 for v in found.values()), (kernel, found)
