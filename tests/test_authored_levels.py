"""Authored levels and pinning (include/crafter_b200.h, cr_author_levels / cr_pin_levels) on the product's kernels on
the SIMT emulator (tests/simt/simt_authored.cpp).

1. The validator accepts the generated worlds of hundreds of seeds, and authoring the world a row decodes to, under
   the same seed, reproduces the row byte for byte; only the authored bit differs.
2. A batch of level -1, fixed, sampled and pinned envs plays on authored copies of the generated rows exactly what it
   plays on the generated rows, in every output and every state buffer, across auto-resets and all three kinds of
   step.
3. Pinning to entry e equals set_levels(seeds[e]), with and without the cache; a weight-0 entry can be pinned and is
   never drawn; an entry at or beyond *n raises the level-table error bit and plays the reference world.
4. Worlds the generator never makes play, step by step, what the C oracle plays on a fresh world of the entry's seed
   with the authored terrain and creatures substituted.
5. Every status bit is raised by a world built to trigger it, and a rejected call changes no row.
6. Staleness as documented; a seed rewritten after authoring is generated over the row by the next fill.
7. The ABI is extended, not changed; the new kernels, k_seed and k_wg_obj do not spill."""
import ctypes

import numpy as np
import pytest
import torch

from crafter_b200 import _cabi
from crafter_b200 import state as state_lib
from crafter_b200 import vector
from crafter_b200.env import AUTHOR_REASONS, LEVEL_PINNED_BASE, LEVEL_SAMPLED, pack_worlds
from tests import hostsim_env
from tests import oracle_levels
from tests.test_build_properties import ptxas  # noqa: F401  (fixture)
from tests.test_level_cache import SimtCacheEnv, simt_cache_lib
from tests.test_levels import KINDS, PS, OracleLevels, Run, world_seed

ERR_LEVEL_TABLE = 4
WATER, GRASS, STONE, PATH, SAND, TREE, LAVA, COAL, IRON, DIAMOND, TABLE, FURNACE = range(1, 13)
COW, ZOMBIE, SKELETON = 1, 2, 3
ODD = dict(area=(37, 29), view=(7, 9), size=(35, 45))
_LIB = []


def simt_authored_lib():
  """tests/simt/simt_authored.cpp: the cache build plus hs_author_levels and hs_pin_levels."""
  if not _LIB:
    here = hostsim_env.HERE
    src = here / 'simt' / 'simt_authored.cpp'
    out = here / 'simt' / '_build' / 'libsimt_authored.so'
    deps = [src] + [here / 'simt' / n for n in ('simt_level_cache.cpp', 'simt_level_sampler.cpp', 'simt_levels.cpp',
                                                 'simt_symbolic.cpp', 'simt_local.cpp', 'simt_env.cpp', 'simt.h')] + list(
        (here.parent / 'crafter_b200' / 'csrc').glob('*.h')) + [here.parent / 'include' / 'crafter_b200.h']
    hostsim_env._compile(out, src, deps)
    L = ctypes.CDLL(str(out))
    base = simt_cache_lib()
    for name in ('hs_create', 'hs_destroy', 'hs_reset', 'hs_step', 'hs_render', 'hs_semantic', 'hs_step_local',
                 'hs_local', 'hs_set_final_local', 'hs_step_symbolic', 'hs_symbolic', 'hs_set_final_symbolic',
                 'hs_set_level_buffers', 'hs_set_levels', 'hs_set_level_table', 'hs_sample_levels', 'hs_seed_only',
                 'hs_set_level_cache', 'hs_fill_level_cache'):
      getattr(L, name).argtypes = getattr(base, name).argtypes
    L.hs_last_error.restype = ctypes.c_char_p
    L.hs_simt_blocks.restype = ctypes.c_long
    L.hs_author_levels.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_int, ctypes.c_void_p]
    L.hs_pin_levels.argtypes = [ctypes.c_void_p] * 3
    _LIB.append(L)
  return _LIB[0]


def pack(materials, creatures=None):
  """(k, W, H) numpy ids -> the (k, W * H) bytes of cr_author_levels, through Env.author_levels' own packing."""
  m = torch.from_numpy(np.asarray(materials, np.int64))
  c = None if creatures is None else torch.from_numpy(np.asarray(creatures, np.int64))
  return pack_worlds(m, c, tuple(m.shape[1:])).numpy()


class SimtAuthoredEnv(SimtCacheEnv):
  """SimtCacheEnv with cr_author_levels and cr_pin_levels on its caller-owned numpy buffers."""

  @staticmethod
  def _load(max_obj_tiles):
    assert max_obj_tiles is None
    return simt_authored_lib()

  def author(self, entries, worlds):
    """cr_author_levels with packed worlds (k, W * H); returns the status words."""
    e = np.ascontiguousarray(entries, np.int32)
    w = np.ascontiguousarray(worlds, np.uint8).reshape(len(e), -1)
    status = np.full(len(e), -7, np.int32)
    self._check(self._L.hs_author_levels(self.h, e.ctypes.data, w.ctypes.data, len(e), status.ctypes.data))
    return status

  def pin_levels(self, entries, mask=None):
    e = np.ascontiguousarray(entries, np.int32)
    m = None if mask is None else np.ascontiguousarray(mask, np.uint8)
    self._check(self._L.hs_pin_levels(self.h, None if m is None else m.ctypes.data, e.ctypes.data))

  def decode(self, rows):
    """(materials, creatures) (k, W, H) of cache rows, as Env.level_worlds decodes them."""
    W, H = self.area
    ents = self.c_ents.view(state_lib.ENT_DTYPE)
    mats, cres = [], []
    for r in rows:
      cre = np.zeros(W * H, np.uint8)
      for e in ents[r, 2:self.c_meta[r, 0]]:
        if 2 <= e['type'] <= 4:
          cre[int(e['x']) * H + int(e['y'])] = e['type'] - 1
      mats.append((self.c_mat[r] & 15).reshape(W, H))
      cres.append(cre.reshape(W, H))
    return np.array(mats), np.array(cres)

  def rows(self):
    return [a.copy() for a in (self.c_mat, self.c_ents, self.c_meta, self.c_tag)]


def oracle_packed(seeds, geometry):
  """The generated worlds of `seeds` from the C oracle, packed as cr_author_levels takes them."""
  key = oracle_levels._key(geometry)
  area = tuple(geometry.get('area', (64, 64)))
  mats, cres = [], []
  for s in seeds:
    st = oracle_levels.fresh_world(int(s), key)
    cre = np.zeros(area, np.int64)
    for t, x, y, *_ in st['objs'][1:]:
      cre[x, y] = t - 1
    mats.append(st['mat'])
    cres.append(cre)
  return pack(mats, cres)


# ---- 1. the validator and the rows --------------------------------------------------------------------------
@pytest.mark.parametrize('geometry', [dict(), ODD], ids=['default', 'odd_area'])
def test_generated_worlds_pass_and_authoring_them_reproduces_the_rows(geometry):
  seeds = np.random.RandomState(7).randint(0, 2 ** 31 - 1, 300).astype(np.int64)
  seeds[:3] = [0, 2 ** 31 - 2, 12345]
  env = SimtAuthoredEnv(num_envs=1, seed=0, **geometry)
  env.set_level_table(seeds)
  env.set_level_cache()
  status = env.author(np.arange(len(seeds)), oracle_packed(seeds, geometry))
  assert (status == 0).all(), np.flatnonzero(status)
  # the authored rows are the oracle's worlds: terrain, creature records in slot order, n
  key, area = oracle_levels._key(geometry), env.area
  ents = env.c_ents.view(state_lib.ENT_DTYPE)
  for i, s in enumerate(seeds):
    want = oracle_levels.fresh_world(int(s), key)
    assert env.c_tag[i] == s and (env.c_mat[i].reshape(area) == want['mat']).all(), i
    creatures = want['objs'][1:]
    n, valid = env.c_meta[i]
    assert n == 2 + len(creatures) and valid == 1 | 4, (i, n, valid)
    got = np.array([[e['type'], e['x'], e['y'], e['health'], e['aux'] if e['type'] != 2 else 0, 0]
                    for e in ents[i, 2:n]], np.int64).reshape(-1, 6)
    assert (got == creatures).all(), i
  # and byte for byte the rows the fill generates, for a few of them
  few = seeds[:6]
  gen = SimtAuthoredEnv(num_envs=1, seed=0, **geometry)
  gen.set_level_table(few)
  gen.set_level_cache()
  gen.fill()
  auth = SimtAuthoredEnv(num_envs=1, seed=0, **geometry)
  auth.set_level_table(few)
  auth.set_level_cache()
  assert (auth.author(np.arange(6), pack(*gen.decode(range(6)))) == 0).all()
  assert (auth.c_mat == gen.c_mat).all() and (auth.c_tag == gen.c_tag).all()
  assert (auth.c_meta[:, 0] == gen.c_meta[:, 0]).all() and (auth.c_meta[:, 1] == gen.c_meta[:, 1] | 4).all()
  for i in range(6):
    n = gen.c_meta[i, 0]
    assert (auth.c_ents[i, 2:n] == gen.c_ents[i, 2:n]).all(), i


# ---- 2. authored copies play what the generated rows play ------------------------------------------------------
class Pair:
  """The same batch twice: `gen` on generated rows, `auth` on authored copies of them; compared after every call."""

  def __init__(self, K, seed, length, **geometry):
    make = lambda: SimtAuthoredEnv(num_envs=K, seed=seed, length=length, auto_reset=True, **geometry)
    self.gen, self.auth = make(), make()

  def both(self, fn):
    return fn(self.gen), fn(self.auth)

  def check(self, where):
    a, b = self.gen, self.auth
    for k, v in a.state.items():
      assert (v == b.state[k]).all(), (where, k, np.flatnonzero((v != b.state[k]).reshape(len(v), -1).any(1)))
    for name in ('final_world_seed', 'level', 'final_semantic', 'final_local', 'final_symbolic', 'final_obs', 'obs'):
      x, y = getattr(a, name), getattr(b, name)
      assert (x is None) == (y is None) and (x is None or (x == y).all()), (where, name)


@pytest.mark.parametrize('geometry', [dict(), ODD], ids=['default', 'odd_area'])
def test_authored_copies_play_what_the_generated_rows_play(geometry):
  K, seed, length = 13, 23, 3
  pair = Pair(K, seed, length, **geometry)
  table = np.array([5, 1234567, 2 ** 31 - 2, 0, 99, 31337], np.int64)
  pair.both(lambda e: e.set_level_table(table, [3, 1, 2, 0, 2, 1], cap=len(table) + 2))
  pair.both(lambda e: e.set_level_cache())
  pair.gen.fill()
  status = pair.auth.author(np.arange(len(table)), pack(*pair.gen.decode(range(len(table)))))
  assert (status == 0).all() and (pair.auth.c_meta[:len(table), 1] & 4).all()
  kind = np.arange(K) % 4
  pair.both(lambda e: e.set_levels(1000 + np.arange(K), kind == 1))
  pair.both(lambda e: e.sample_levels(kind == 2))
  pinned = np.arange(K) % len(table)
  pair.both(lambda e: e.pin_levels(pinned, kind == 3))
  pair.both(lambda e: e.reset())
  pair.check('reset')
  assert (pair.auth.level[kind == 3] == LEVEL_PINNED_BASE - pinned[kind == 3]).all()
  rs = np.random.RandomState(seed)
  episodes = np.zeros(K, int)
  for t in range(12):
    actions = rs.randint(0, 17, K).astype(np.int32)
    ra, rb = pair.both(lambda e: [x.copy() for x in e.step(actions, KINDS[t % 3])])
    for x, y in zip(ra, rb):
      assert (x == y).all(), t
    pair.check(t)
    episodes += rb[2].astype(bool)
    rows = pair.auth.cached_rows()
    assert (rows[kind == 3] == pinned[kind == 3]).all(), 'a pinned env was not served its entry\'s row'
  assert (episodes >= 3).all(), episodes
  assert set(pair.auth.final_world_seed[kind == 3].tolist()) <= set(table.tolist())


# ---- 3. pinning --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('cache', [False, True], ids=['generated', 'cached'])
def test_pinning_equals_set_levels_of_the_entrys_seed(cache):
  K, seed, length = 7, 41, 3
  table = np.array([77, 2 ** 31 - 2, 5, 424242], np.int64)
  entries = np.array([0, 1, 2, 3, 1, 2, 0], np.int32)
  pin = SimtAuthoredEnv(num_envs=K, seed=seed, length=length, auto_reset=True)
  lev = SimtAuthoredEnv(num_envs=K, seed=seed, length=length, auto_reset=True)
  pin.set_level_table(table, [1, 0, 1, 1])  # entry 1 has weight 0: pinnable all the same
  if cache:
    pin.set_level_cache()
    pin.fill()
  pin.pin_levels(entries)
  lev.set_levels(table[entries].astype(np.int32))
  pin.reset()
  lev.reset()
  rs = np.random.RandomState(seed)
  for t in range(10):
    actions = rs.randint(0, 17, K).astype(np.int32)
    ra = [x.copy() for x in pin.step(actions, KINDS[t % 3])]
    rb = [x.copy() for x in lev.step(actions, KINDS[t % 3])]
    for x, y in zip(ra, rb):
      assert (x == y).all(), t
    for k, v in pin.state.items():
      assert (v == lev.state[k]).all(), (t, k)
    assert (pin.final_world_seed == lev.final_world_seed).all()
    if cache:
      assert (pin.cached_rows() == entries).all()
  assert (pin.level == LEVEL_PINNED_BASE - entries).all() and (pin.errors() == 0).all()


def test_a_zero_weight_entry_is_pinned_but_never_drawn():
  K, seed = 9, 3
  env = SimtAuthoredEnv(num_envs=K, seed=seed, length=2, auto_reset=True)
  table = np.array([11, 22, 33], np.int64)
  env.set_level_table(table, [1, 0, 1])
  env.set_level_cache()
  env.fill()
  env.sample_levels(np.arange(K) != 0)
  env.pin_levels(np.ones(K, np.int32), np.arange(K) == 0)
  env.reset()
  drawn = set()
  for t in range(12):
    env.step(np.zeros(K, np.int32), 'semantic')
    ws = env.world_seed()
    assert ws[0] == 22
    drawn |= set(ws[1:].tolist())
  assert drawn == {11, 33}, drawn
  assert env.level[0] == LEVEL_PINNED_BASE - 1 and (env.level[1:] == LEVEL_SAMPLED).all()


def test_an_entry_beyond_n_raises_the_error_bit_and_plays_the_reference_world():
  K, seed = 3, 12
  env = SimtAuthoredEnv(num_envs=K, seed=seed, length=2, auto_reset=True)
  env.set_level_table([7, 8], cap=6)
  env.pin_levels(np.array([1, 4, -5], np.int32))  # entry 4 lies beyond *n = 2; a negative entry is none at all
  env.reset()
  assert env.errors().tolist() == [0, ERR_LEVEL_TABLE, ERR_LEVEL_TABLE]
  ws = env.world_seed()
  assert ws[0] == 8 and ws[1] == world_seed(seed + 1, 1) and ws[2] == world_seed(seed + 2, 1)
  assert env.level.tolist() == [-4, -7, -(2 ** 31)]


def test_pinning_needs_a_table_and_the_level_buffer():
  env = SimtAuthoredEnv(num_envs=2, seed=1)
  with pytest.raises(RuntimeError, match='no level table'):
    env.pin_levels(np.zeros(2, np.int32))
  bare = SimtAuthoredEnv(num_envs=2, seed=1, level_buffers=False)
  bare.set_level_table([3])
  with pytest.raises(RuntimeError, match='no level buffer'):
    bare.pin_levels(np.zeros(2, np.int32))


# ---- 4. worlds the generator never makes, against the C oracle ----------------------------------------------------
def blank(material, area=(64, 64)):
  return np.full(area, material, np.int64), np.zeros(area, np.int64)


def probe_worlds(capacity, area=(64, 64)):
  """{name: (materials, creatures)}: worlds the generator never makes; the start is (W/2, H/2) = (32, 32)."""
  W, H = area
  px, py = W // 2, H // 2
  out = {}
  m, c = blank(GRASS)
  m[px - 1, py] = m[px + 1, py] = m[px, py - 1] = LAVA
  m[px + 3:px + 6, :] = STONE
  out['lava_beside_start'] = (m, c)
  m, c = blank(GRASS)
  m[px, py + 1], m[px + 1, py + 1], m[px - 1, py - 1], m[px, py - 1] = COAL, IRON, DIAMOND, TABLE
  m[px - 1, py], m[px + 1, py], m[px, py + 2], m[px + 2, py] = FURNACE, TREE, WATER, STONE
  out['ores_table_furnace_within_reach'] = (m, c)
  m, c = blank(GRASS)
  c[px + 1, py] = c[px, py + 1] = c[px - 1, py] = ZOMBIE
  c[px + 7, py + 7] = COW
  out['zombies_next_to_the_player'] = (m, c)
  m, c = blank(SAND)
  m[px:, :] = PATH
  for x, y in ((px - 3, py), (px + 2, py + 1), (5, 5), (60, 60), (px + 1, py - 4)):
    c[x, y] = COW
  out['cows_on_sand_and_path'] = (m, c)
  m, c = blank(STONE)
  m[:, py] = PATH
  m[px, :] = PATH
  for x in (3, 10, 20, 45, 58):
    c[x, py] = SKELETON
  c[px, 50] = SKELETON
  out['skeletons_on_path_without_tunnels'] = (m, c)
  m, c = blank(SAND)
  m[10:20, 10:20], m[40:50, 5:15], m[px + 2:px + 4, :] = WATER, STONE, TREE
  c[px - 5, py - 5] = ZOMBIE
  out['no_grass'] = (m, c)
  m, c = blank(PATH)
  c[px + 4, py], c[10, 10] = SKELETON, ZOMBIE
  out['all_path'] = (m, c)
  m, c = blank(WATER)
  m[px, py] = GRASS
  out['water_everywhere_but_the_start'] = (m, c)
  m, c = blank(SAND)  # no grass and no path: balance spawns nothing, so the arena stays exactly full
  cells = [(x, y) for x in range(W) for y in range(H) if (x, y) != (px, py)]
  for x, y in cells[::7][:capacity - 2]:
    c[x, y] = COW
  out['slot_capacity_minus_two_creatures'] = (m, c)
  return out


def authored_state(mat, cre, ws, key, ncy):
  """The oracle's fresh state of world seed `ws` with the authored terrain and creatures substituted."""
  base = oracle_levels.fresh_world(int(ws), key)
  player = base['objs'][0]
  rows = [player]
  for x, y in zip(*np.nonzero(cre)):  # x-major cell order, the slot order of k_wg_obj
    t = int(cre[x, y]) + 1
    rows.append([t, x, y, 5 if t == 3 else 3, 0, 0])
  touched = sorted({(int(r[1]) // 12) * ncy + int(r[2]) // 12 for r in rows})
  return dict(mat=np.asarray(mat, np.uint8), objs=np.array(rows, np.int32), player=base['player'],
              touched=np.array(touched, np.int32))


class AuthoredLevelEnv(oracle_levels.LevelEnv):
  """An oracle LevelEnv that plays table entries: level -3 - e starts each episode on entry e, authored or not."""

  def __init__(self, table, worlds, seed=0, **kwargs):
    super().__init__(seed=seed, **kwargs)
    self.table, self.worlds = table, worlds
    area = kwargs.get('area', (64, 64))
    self.ncy = (area[1] + 11) // 12

  def reset(self):
    if self.level > LEVEL_PINNED_BASE:
      return super().reset()
    e = LEVEL_PINNED_BASE - self.level
    self.episode += 1
    self.world_seed = int(self.table[e])
    if e in self.worlds:
      st = authored_state(*self.worlds[e], self.world_seed, self._geometry, self.ncy)
    else:
      st = oracle_levels.fresh_world(self.world_seed, self._geometry)
    self.env.import_state(st, 0, self.episode, self.world_seed)
    return self.env.render()


class AuthoredRun(Run):
  """tests/test_levels.Run with a SimtAuthoredEnv beside AuthoredLevelEnv oracles."""

  def __init__(self, K, seed, length, start_step, table, worlds):
    self.env = SimtAuthoredEnv(num_envs=K, seed=seed, length=length, auto_reset=True)
    self.ora = OracleLevels(0, seed)
    self.ora.refs = [AuthoredLevelEnv(table, worlds, seed=seed + i, length=length) for i in range(K)]
    self.K, self.grid, self.start_step = K, self.env.grid, start_step
    self.reached = dict(episodes=0, terminal=0, night=0, kinds=set(), seeds=set())
    self.rs = np.random.RandomState(seed)

  def pin_levels(self, entries):
    self.env.pin_levels(entries)
    self.ora.set_levels(LEVEL_PINNED_BASE - np.asarray(entries, np.int64))


@pytest.mark.parametrize('length, start', [(4, None), (160, 155)], ids=['day', 'nightfall_and_balance'])
def test_authored_worlds_play_what_the_oracle_plays(length, start):
  probe = SimtAuthoredEnv(num_envs=1, seed=0)
  worlds = list(probe_worlds(probe.capacity).values())
  table = np.array([1000 + 17 * i for i in range(len(worlds))] + [31337], np.int64)  # the last entry: generated
  K, seed = len(table) + 1, 70
  run = AuthoredRun(K, seed, length, start, table, dict(enumerate(worlds)))
  run.env.set_level_table(table)
  run.env.set_level_cache()
  run.env.fill()
  status = run.env.author(np.arange(len(worlds)), pack([m for m, _ in worlds], [c for _, c in worlds]))
  assert (status == 0).all(), status
  run.pin_levels(np.arange(K) % len(table))
  run.reset()
  for t in range(14):
    run.step(t, KINDS[t % 3])
  r = run.reached
  assert r['kinds'] == set(KINDS) and r['episodes'] >= 2 * K, r
  assert set(table.tolist()) <= r['seeds'], r['seeds']
  if start is not None:
    assert r['night'] > 0, r
  assert (run.env.errors() == 0).all()


# ---- 5. rejections -------------------------------------------------------------------------------------------------
def test_every_status_bit_is_raised_and_a_rejected_call_changes_no_row():
  env = SimtAuthoredEnv(num_envs=2, seed=4)
  table = np.array([3, 4, 5, 6], np.int64)
  env.set_level_table(table)
  env.set_level_cache()
  env.fill()
  cap = env.capacity
  good = blank(GRASS)
  bad = {}
  m, c = blank(GRASS)
  m[3, 3] = 0
  bad[1] = (m, c)  # material 0
  m, c = blank(GRASS)
  m[5, 5], c[5, 5] = STONE, COW
  bad[2] = (m, c)  # a creature on stone
  m, c = blank(GRASS)
  m[32, 32] = WATER
  bad[4] = (m, c)  # the start on water
  m, c = blank(GRASS)
  c.reshape(-1)[:cap - 1] = COW  # one creature too many (the start, cell 32 * 64 + 32, lies beyond them)
  bad[8] = (m, c)
  before = env.rows()
  for bit, (m, c) in bad.items():
    status = env.author([0, 1], pack([good[0], m], [good[1], c]))
    assert status.tolist() == [0, bit], (bit, status)
  m, c = blank(GRASS)
  c[32, 32] = ZOMBIE
  assert env.author([2], pack([m], [c])).tolist() == [4]  # a creature on the start
  g = pack([good[0]], [good[1]])[0]
  raw = g.copy()
  raw[7] = GRASS | 0x40  # bit 6 set
  assert env.author([0], raw[None]).tolist() == [1]
  raw[7] = 13  # a material above 12
  assert env.author([0], raw[None]).tolist() == [1]
  assert env.author([4, -1], np.stack([g, g])).tolist() == [16, 16]  # outside [0, capacity)
  full = pack([bad[8][0]], [bad[8][1]])[0]
  assert env.author([1, 2, 1, 1], np.stack([g, g, g, full])).tolist() == [16, 0, 16, 16 | 8]  # more than once
  after = env.rows()
  assert all((a == b).all() for a, b in zip(before, after)), 'a rejected call changed a row'
  # the claims were released: the same entries are accepted in the next call
  assert env.author([1, 2], np.stack([g, g])).tolist() == [0, 0]
  assert (env.c_meta[[1, 2], 1] == 5).all() and (env.c_tag[[1, 2]] == [4, 5]).all()
  assert (env.c_mat[0] == before[0][0]).all() and (env.c_mat[3] == before[0][3]).all()


def test_authoring_needs_a_table_and_a_cache():
  env = SimtAuthoredEnv(num_envs=1, seed=0)
  g = pack(*map(lambda a: a[None], blank(GRASS)))
  with pytest.raises(RuntimeError, match='no level table'):
    env.author([0], g)
  env.set_level_table([9])
  with pytest.raises(RuntimeError, match='no level cache'):
    env.author([0], g)
  env.set_level_cache()
  assert env.author([0], g).tolist() == [0]


# ---- 6. staleness --------------------------------------------------------------------------------------------------
def marked(material):
  """A grass world with `material` at cell (0, 0), far from anything the player can change in a short episode."""
  m, c = blank(GRASS)
  m[0, 0] = material
  return pack(m[None], c[None])


def test_a_reauthored_entry_reaches_a_pinned_env_by_its_second_new_episode():
  K = 2
  env = SimtAuthoredEnv(num_envs=K, seed=9, length=3, auto_reset=True)
  env.set_level_table([50, 60])
  env.set_level_cache()
  assert env.author([0], marked(DIAMOND)).tolist() == [0]
  env.pin_levels(np.zeros(K, np.int32))
  env.reset()
  plays = lambda: env.state['mat'].reshape(K, -1)[:, 0].tolist()
  assert plays() == [DIAMOND] * K
  for _ in range(4):
    env.step(np.zeros(K, np.int32))
  assert env.author([0], marked(TABLE)).tolist() == [0]  # mid-episode
  seen = []
  while len(seen) < 2:
    _, _, done = env.step(np.zeros(K, np.int32))
    if done.any():
      assert done.all()
      seen.append(plays())
  assert seen[1] == [TABLE] * K, seen  # the first new episode may still play the old world
  # pinning again makes a re-authored entry hold from the very next episode
  for _ in range(1):
    env.step(np.zeros(K, np.int32))
  assert env.author([0], marked(FURNACE)).tolist() == [0]
  env.pin_levels(np.zeros(K, np.int32))
  while True:
    _, _, done = env.step(np.zeros(K, np.int32))
    if done.any():
      assert plays() == [FURNACE] * K
      break
  assert (env.world_seed() == 50).all()


def test_a_rewritten_seed_is_generated_over_an_authored_row_by_the_next_fill():
  env = SimtAuthoredEnv(num_envs=1, seed=0)
  env.set_level_table([50, 60])
  env.set_level_cache()
  env.fill()
  assert env.author([0, 1], np.concatenate([marked(DIAMOND), marked(TABLE)])).tolist() == [0, 0]
  env.fill()  # the seeds stand: the authored rows survive
  assert (env.c_meta[:, 1] & 4).all() and env.c_mat[0, 0] == DIAMOND
  env.t_seeds[0] = 777
  env.fill()
  fresh = SimtAuthoredEnv(num_envs=1, seed=0)
  fresh.set_level_table([777])
  fresh.set_level_cache()
  fresh.fill()
  assert env.c_tag.tolist() == [777, 60] and env.c_meta[0, 1] & 4 == 0 and env.c_meta[1, 1] & 4
  assert (env.c_mat[0] == fresh.c_mat[0]).all() and (env.c_meta[0] == fresh.c_meta[0]).all()


# ---- host side, ABI, build ---------------------------------------------------------------------------------------
def test_pack_worlds_checks_shapes_and_dtypes_and_flags_bad_values():
  m = np.full((2, 4, 3), GRASS, np.int64)
  c = np.zeros((2, 4, 3), np.int64)
  c[1, 2, 1] = SKELETON
  w = pack_worlds(m, c, (4, 3))
  assert w.dtype == torch.uint8 and tuple(w.shape) == (2, 12) and int(w[1, 2 * 3 + 1]) == GRASS | SKELETON << 4
  m[0, 0, 0], c[0, 1, 1] = 13, 4
  w = pack_worlds(m, c, (4, 3))
  assert int(w[0, 0]) == 0xC0 and int(w[0, 4]) == 0xC0
  with pytest.raises(ValueError, match='shape'):
    pack_worlds(m, None, (3, 4))
  with pytest.raises(ValueError, match='integers'):
    pack_worlds(m.astype(np.float32), None, (4, 3))
  with pytest.raises(ValueError, match='shape of materials'):
    pack_worlds(m, c[:1], (4, 3))
  assert [bit for bit, _ in AUTHOR_REASONS] == [1, 2, 4, 8, 16]


def test_vector_env_passes_authoring_and_pinning_through():
  calls = []

  class FakeEnv:

    def author_levels(self, entries, materials, creatures=None):
      calls.append(('author', entries, creatures))

    def level_worlds(self, entries):
      calls.append(('worlds', entries))
      return 'w'

    def pin_levels(self, entries, mask=None):
      calls.append(('pin', entries, mask))

  venv = vector.VectorEnv.__new__(vector.VectorEnv)
  venv.env = FakeEnv()
  venv.author_levels([1], 'm')
  assert venv.level_worlds([2]) == 'w'
  venv.pin_levels([0, 1], [True, False])
  assert calls == [('author', [1], None), ('worlds', [2]), ('pin', [0, 1], [True, False])]


def test_abi_is_extended_not_changed():
  names = [f[0] for f in _cabi.CrState._fields_]
  assert len(names) == 24 and _cabi.ABI_VERSION == 6
  assert {'cr_author_levels', 'cr_pin_levels'} <= set(_cabi.EXPORTS)
  header = (hostsim_env.HERE.parent / 'include' / 'crafter_b200.h').read_text()
  assert 'int cr_author_levels(' in header and 'int cr_pin_levels(' in header
  assert '#define CR_LEVEL_PINNED(e) (-3 - (e))' in header and '#define CR_ABI_VERSION 6' in header
  assert PS['world_seed'] == 11


def test_authoring_kernels_do_not_spill(ptxas):  # noqa: F811
  for kernel in ('k_author_check', 'k_author_copy', 'k_author_tag', 'k_pin_levels', 'k_seed', 'k_wg_obj'):
    found = {targs: v for (name, targs), v in ptxas.items() if name == kernel}
    assert found and all(v.get('spill', 0) == 0 for v in found.values()), (kernel, found)
