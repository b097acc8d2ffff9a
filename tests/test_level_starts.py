"""Level starts (include/crafter_b200.h, cr_set_level_starts) on the product's kernels on the SIMT emulator
(tests/simt/simt_level_starts.cpp), against the C oracle.

The restatement never reads the start notes.  It decides each episode's entry as tests/test_level_stats.py does
(`restated_entry` for a sampled env, the pinned entry below *n) and takes the start of that entry from the start table
as it stands when the entry is decided.  An episode then starts, on the oracle, from the canonical fresh state of its
world (tests/oracle_levels.fresh_world, or the authored world substituted into it) with the player row edited when the
start is on and applicable: x, y, facing, inventory and both last healths, and the touched chunks recomputed from the
objects.  The oracle imports that state and steps it with the same actions.

1. A batch of level -1, fixed, sampled, pinned (one entry at or beyond *n) and authored envs, with starts holding tools
   and resources, low food or health, every facing and off-centre positions, plays what the oracle plays: observations,
   reward, done and the canonical state at every step, across auto-resets, with and without auto_reset, in all three
   kinds of step, at the default and an odd geometry, with and without the cache.  One entry's start cell is not
   walkable in its world and another's holds a creature: their episodes start at the reference's start and raise
   error bit 8.  A mid-run start rewrite reaches each env when the restatement says, and sample_levels / pin_levels
   make it hold from the next episode.
2. An all-zero start table gives a batch identical to one without starts, in all of cr_state, after every call.
3. A snapshot of the state and the notes continues, in a fresh env, with the same starts.
4. Goal plus start: goal collect_stone with a wood pickaxe next to stone is reached, pays 1.0 and ends the episode.
5. level_start, host validation, the vector env's pass-through, the ABI, and the kernels' register budget."""
import ctypes

import numpy as np
import pytest
import torch

from crafter_b200 import _cabi
from crafter_b200 import rules
from crafter_b200 import vector
from crafter_b200.env import ERR_LEVEL_START, START_WORDS, Env, goal_mask, level_start
from oracle import canon
from oracle import oracle_env
from tests import hostsim_env
from tests import oracle_levels
from tests.test_authored_levels import ODD, authored_state, oracle_packed
from tests.test_build_properties import ptxas  # noqa: F401  (fixture)
from tests.test_level_goals import SimtGoalsEnv, simt_goals_lib
from tests.test_level_stats import Restated
from tests.test_levels import KINDS, PS, expected_obs, obs_problem, world_seed

WATER, GRASS, STONE, PATH, SAND = 1, 2, 3, 4, 5
WALKABLE = (GRASS, SAND, PATH)
# the canonical player vector (oracle/canon.py): inventory 0..15, achievements 16..37, then these
P_FACING, P_LAST_HEALTH, P_X, P_Y, P_ENV_LAST_HEALTH = 43, 44, 45, 46, 47
_LIB = []


def simt_starts_lib():
  """tests/simt/simt_level_starts.cpp: the goals build plus hs_set_level_starts."""
  if not _LIB:
    here = hostsim_env.HERE
    src = here / 'simt' / 'simt_level_starts.cpp'
    out = here / 'simt' / '_build' / 'libsimt_level_starts.so'
    deps = [src] + [here / 'simt' / n for n in (
        'simt_level_goals.cpp', 'simt_level_stats.cpp', 'simt_authored.cpp', 'simt_level_cache.cpp',
        'simt_level_sampler.cpp', 'simt_levels.cpp', 'simt_symbolic.cpp', 'simt_local.cpp', 'simt_env.cpp', 'simt.h')] + list(
            (here.parent / 'crafter_b200' / 'csrc').glob('*.h')) + [here.parent / 'include' / 'crafter_b200.h']
    hostsim_env._compile(out, src, deps)
    L = ctypes.CDLL(str(out))
    base = simt_goals_lib()
    for name in ('hs_create', 'hs_destroy', 'hs_reset', 'hs_step', 'hs_render', 'hs_semantic', 'hs_step_local',
                 'hs_local', 'hs_set_final_local', 'hs_step_symbolic', 'hs_symbolic', 'hs_set_final_symbolic',
                 'hs_set_level_buffers', 'hs_set_levels', 'hs_set_level_table', 'hs_sample_levels', 'hs_seed_only',
                 'hs_set_level_cache', 'hs_fill_level_cache', 'hs_author_levels', 'hs_pin_levels',
                 'hs_set_level_stats', 'hs_set_level_goals'):
      getattr(L, name).argtypes = getattr(base, name).argtypes
    L.hs_last_error.restype = ctypes.c_char_p
    L.hs_simt_blocks.restype = ctypes.c_long
    L.hs_set_level_starts.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_int]
    _LIB.append(L)
  return _LIB[0]


class SimtStartsEnv(SimtGoalsEnv):
  """SimtGoalsEnv with the start table and the start notes in caller-owned numpy buffers."""

  starts = start_notes = None

  @staticmethod
  def _load(max_obj_tiles):
    assert max_obj_tiles is None
    return simt_starts_lib()

  def set_level_starts(self, starts, cap=None):
    """Register `starts` (padded with zero records to `cap`, None: the table's capacity) and notes filled with 0."""
    cap = cap or self.t_cap
    self.starts = np.zeros((cap, START_WORDS), np.int32)
    self.starts[:len(starts)] = starts
    self.start_notes = np.zeros((self.B, 4, START_WORDS), np.int32)
    self._check(self._L.hs_set_level_starts(self.h, self.starts.ctypes.data, self.start_notes.ctypes.data, cap))

  def remove_level_starts(self):
    self._check(self._L.hs_set_level_starts(self.h, None, None, 0))


# ---- the restatement ---------------------------------------------------------------------------------------------
def applicable(st, start, area):
  """Whether an `on` start record can place the player in the fresh canonical state `st`."""
  W, H = area
  x, y, facing = (int(v) for v in start[1:4])
  inv = np.asarray(start[4:])
  if not (0 <= x < W and 0 <= y < H and 0 <= facing < 4 and (inv >= 0).all() and (inv <= 9).all() and inv[0] >= 1):
    return False
  creatures = st['objs'][1:]
  return int(st['mat'][x, y]) in WALKABLE and not ((creatures[:, 1] == x) & (creatures[:, 2] == y)).any()


def started_state(st, start, ncy):
  """The fresh canonical state `st` with the player at the start: its row in objs and in player, and touched."""
  objs, player = st['objs'].copy(), st['player'].copy()
  x, y, facing = (int(v) for v in start[1:4])
  inv = np.asarray(start[4:], np.int64)
  objs[0, 1:5] = x, y, inv[0], facing
  player[:16] = inv
  player[P_FACING], player[P_LAST_HEALTH], player[P_ENV_LAST_HEALTH] = facing, inv[0], inv[0]
  player[P_X], player[P_Y] = x, y
  touched = sorted({(int(r[1]) // 12) * ncy + int(r[2]) // 12 for r in objs})
  return dict(mat=st['mat'], objs=objs, player=player, touched=np.array(touched, np.int32))


class StartRestated(Restated):
  """Restated (tests/test_level_stats.py) plus the world seed and the start of every decided episode, the start taken
  from `env.starts` (rewritten in place by the tests) when its entry is decided."""

  def __init__(self, env, seed):
    super().__init__(env, seed, 1)
    self.ws = [{} for _ in range(env.B)]
    self.start = [{} for _ in range(env.B)]

  def _decide(self, i, e):
    if e in self.decided[i]:
      return
    super()._decide(i, e)
    r, level = self.decided[i][e], int(self.env.level[i])
    seeds, _ = self.env.table()
    self.ws[i][e] = int(seeds[r]) if r >= 0 else level if level >= 0 else world_seed(self.seed + i, e)
    starts = self.env.starts
    self.start[i][e] = starts[r].copy() if starts is not None and 0 <= r < len(starts) else np.zeros(START_WORDS, np.int32)

  def check_notes(self, where):
    ep = self.env.episodes()
    for i in range(self.env.B):
      for e in range(ep[i], ep[i] + 3):
        if e in self.start[i]:
          assert (self.env.start_notes[i, e & 3] == self.start[i][e]).all(), (where, i, e, self.env.start_notes[i])


class StartRun:
  """A SimtStartsEnv beside one C oracle env per env, compared after every call: reward, done, the observation of the
  step kind and the canonical state; the terminal semantic map of the envs that finished; the start notes; error
  bit 8 of every env."""

  def __init__(self, K, seed, length, table, weights, auto_reset, cached, authored=None, **geometry):
    self.env = SimtStartsEnv(num_envs=K, seed=seed, length=length, auto_reset=auto_reset, **geometry)
    self.env.set_level_table(table, weights, cap=len(table) + 2)
    self.authored = {}
    if cached:
      self.env.set_level_cache()
      self.env.fill()
      if authored:  # {entry: world seed}: the generated world of another seed, authored under the entry
        entries = sorted(authored)
        assert (self.env.author(entries, oracle_packed([authored[e] for e in entries], geometry)) == 0).all()
        for e in entries:
          st = oracle_levels.fresh_world(int(authored[e]), oracle_levels._key(geometry))
          cre = np.zeros(st['mat'].shape, np.int64)
          for t, x, y, *_ in st['objs'][1:]:
            cre[x, y] = t - 1
          self.authored[e] = (st['mat'], cre)
    self.K, self.seed, self.auto_reset = K, seed, auto_reset
    self.area = tuple(geometry.get('area', (64, 64)))
    self.ncy = (self.area[1] + 11) // 12
    self.key = oracle_levels._key(geometry)
    self.refs = [oracle_env.OracleEnv(seed=seed + i, length=length, **geometry) for i in range(K)]
    self.res = StartRestated(self.env, seed)
    self.grid = self.env.grid
    self.err = np.zeros(K, bool)
    self.reached = dict(episodes=0, applied=0, refused=0, kinds=set(), facings=set(), authored=0)
    self.rs = np.random.RandomState(seed)

  def relevel(self, fn, mask):
    fn(self.env)
    self.res.relevel(mask)
    self.check('relevel')

  def fresh(self, i):
    """Start env i's oracle on the episode its SIMT env is on now."""
    e = int(self.env.episodes()[i])
    self.res.started(np.arange(self.K) == i)
    ws, r, start = self.res.ws[i][e], self.res.decided[i][e], self.res.start[i][e]
    if r in self.authored:
      st = authored_state(*self.authored[r], ws, self.key, self.ncy)
      self.reached['authored'] += 1
    else:
      st = oracle_levels.fresh_world(ws, self.key)
    if start[0]:
      if applicable(st, start, self.area):
        st = started_state(st, start, self.ncy)
        self.reached['applied'] += 1
        self.reached['facings'].add(int(start[3]))
      else:
        self.err[i] = True
        self.reached['refused'] += 1
    self.refs[i].import_state(st, 0, e, ws)
    self.reached['episodes'] += 1
    return self.refs[i].render()

  def reset(self, mask=None, kind='rgb'):
    obs = self.env.reset(mask, kind=kind).copy()
    for i in range(self.K) if mask is None else np.flatnonzero(mask):
      frame = self.fresh(i)
      problem = obs_problem(kind, obs[i], expected_obs(self.refs[i], kind, frame, self.grid), self.grid)
      assert problem is None, ('reset', kind, i, problem)
    self.check('reset')

  def check(self, where):
    for i, ref in enumerate(self.refs):
      problem = canon.diff(ref.export_state(), self.env.snapshot(i))
      assert problem is None, (where, i, problem)
    assert ((self.env.errors() & ERR_LEVEL_START != 0) == self.err).all(), (where, self.env.errors(), self.err)
    self.res.check_notes(where)

  def step(self, t, kind):
    actions = self.rs.randint(0, 17, self.K).astype(np.int32)
    obs, reward, done = [x.copy() for x in self.env.step(actions, kind)]
    self.reached['kinds'].add(kind)
    for i, ref in enumerate(self.refs):
      where = (t, kind, i)
      frame, r, d = ref.step(int(actions[i])) if kind == 'rgb' else (None,) + ref.step_norender(int(actions[i]))
      assert np.float32(r) == reward[i] and d == bool(done[i]), where + ('reward / done', r, reward[i], d)
      if d and self.auto_reset:
        assert (self.env.final_semantic[i] == ref.semantic()).all(), where + ('terminal semantic',)
        frame = self.fresh(i)
      problem = obs_problem(kind, obs[i], expected_obs(ref, kind, frame, self.grid), self.grid)
      assert problem is None, where + ('obs', problem)
    self.check(t)
    if not self.auto_reset and done.any():  # the caller resets the envs that are done
      self.reset(done, kind=KINDS[(t + 1) % 3])
    return done


def start_table(area, seeds, geometry):
  """Starts for the entries of `seeds`: tools and resources, low food / health, every facing, off-centre positions,
  one entry off; entry 4 starts on a cell of its world that is not walkable and entry 5 on one of its creatures."""
  W, H = area
  cx, cy = W // 2, H // 2
  key = oracle_levels._key(geometry)
  starts = [
      level_start({'wood_pickaxe': 1, 'stone_pickaxe': 1, 'wood': 5, 'stone': 3, 'sapling': 2}, (cx + 2, cy - 1),
                  'right', area),
      level_start({'health': 2, 'food': 1, 'drink': 3}, (cx + 1, cy + 1), 'up', area),
      level_start({'energy': 1, 'coal': 4, 'iron': 2, 'wood_sword': 1}, (cx - 2, cy + 2), 'left', area),
      np.zeros(START_WORDS, np.int32),
  ]
  mat = oracle_levels.fresh_world(int(seeds[4]), key)['mat']
  bad = np.argwhere(mat == WATER)
  bad = bad if len(bad) else np.argwhere(~np.isin(mat, WALKABLE))
  starts.append(level_start({'drink': 1}, tuple(int(v) for v in bad[0]), 'down', area))
  objs = oracle_levels.fresh_world(int(seeds[5]), key)['objs']
  assert len(objs) > 1, 'the entry world has a creature'
  starts.append(level_start({'food': 4}, (int(objs[1][1]), int(objs[1][2])), (0, -1), area))
  starts.append(level_start({'iron_pickaxe': 1, 'health': 5}, (cx, cy), (0, 1), area))  # the centre, other vitals
  return np.array(starts, np.int32)


# ---- 1. a mixed batch against the oracle ---------------------------------------------------------------------------
@pytest.mark.parametrize('auto_reset', [True, False], ids=['auto_reset', 'no_auto_reset'])
@pytest.mark.parametrize('cached', [True, False], ids=['cached', 'uncached'])
@pytest.mark.parametrize('geometry', [dict(), ODD], ids=['default', 'odd_area'])
def test_the_batch_plays_what_the_oracle_plays_from_the_starts(geometry, cached, auto_reset):
  K, seed, length = 14, 61, 9
  table = np.array([5, 1234567, 2 ** 31 - 2, 99, 31337, 4242, 777], np.int64)
  weights = [3, 2, 2, 1, 1, 1, 0]  # entry 6: pinned only
  run = StartRun(K, seed, length, table, weights, auto_reset, cached, authored={2: 77, 6: 78} if cached else None,
                 **geometry)
  area = run.area
  run.env.set_level_starts(start_table(area, table, geometry))
  kind = np.array([0, 1, 2, 3, 4, 4, 0, 1, 2, 3, 4, 4, 2, 4])  # 0: level -1, 1: fixed, 2 and 3: sampled, 4: pinned
  pins = np.zeros(K, np.int32)
  pins[kind == 4] = [6, 9, 5, 4, 0]  # entry 9 lies beyond *n = 7
  run.relevel(lambda e: e.set_levels(1000 + np.arange(K), kind == 1), kind == 1)
  run.relevel(lambda e: e.sample_levels((kind == 2) | (kind == 3)), (kind == 2) | (kind == 3))
  run.relevel(lambda e: e.pin_levels(pins, kind == 4), kind == 4)
  run.reset()
  W, H = area
  for t in range(30):
    if t == 12:  # a rewrite: episodes decided from now on take the new starts, the decided ones keep theirs
      run.env.starts[3] = level_start({'stone': 9}, (W // 2 - 1, H // 2), 'up', area)
      run.env.starts[0, 0] = 0
      run.check('rewrite')
    if t == 20:  # sample_levels / pin_levels decide the next two episodes again: the new starts hold from the next one
      m = np.arange(K) == 2
      run.relevel(lambda e: e.sample_levels(m), m)
      m = np.arange(K) == 5
      run.relevel(lambda e: e.pin_levels(np.full(K, 3, np.int32), m), m)
      e = run.env.episodes()[5] + 1
      assert (run.res.start[5][e] == run.env.starts[3]).all()
    run.step(t, KINDS[t % 3])
  r = run.reached
  assert r['kinds'] == set(KINDS) and r['episodes'] >= 3 * K, r
  assert r['applied'] >= K and r['refused'] >= 2 and r['facings'] == {0, 1, 2, 3}, r
  assert not cached or r['authored'] >= 2, r
  assert run.err[kind == 4].tolist() == [False, False, True, True, False]  # the pins of entries 5 and 4


def test_error_bit_is_clear_without_an_inapplicable_start():
  K, seed = 6, 4
  run = StartRun(K, seed, 5, np.array([10, 20], np.int64), [1, 1], True, False)
  W, H = run.area
  run.env.set_level_starts([level_start({'stone_pickaxe': 1}, (W // 2 + 1, H // 2), 'left'), np.zeros(20, np.int32)])
  run.relevel(lambda e: e.sample_levels(), None)
  run.reset()
  for t in range(12):
    run.step(t, KINDS[t % 3])
  assert run.reached['applied'] > 0 and (run.env.errors() == 0).all()


# ---- 2. an all-zero table is no table ------------------------------------------------------------------------------
def test_all_zero_starts_change_nothing():
  K, seed, length = 12, 5, 6
  table = np.array([7, 8, 9, 10], np.int64)

  def make(starts):
    env = SimtStartsEnv(num_envs=K, seed=seed, length=length, auto_reset=True)
    env.set_level_table(table, [1, 2, 3, 1])
    env.set_level_cache()
    env.fill()
    env.set_level_stats()
    if starts:
      env.set_level_starts(np.zeros((4, START_WORDS), np.int32))
    return env

  a, b = make(True), make(False)
  both = lambda fn: [fn(e) for e in (a, b)]

  def same(where):
    for k, v in a.state.items():
      assert (v == b.state[k]).all(), (where, k)
    for n in ('final_world_seed', 'final_entry', 'stats', 'ring', 'obs', 'final_obs', 'final_local', 'final_symbolic',
              'final_semantic'):
      x, y = getattr(a, n), getattr(b, n)
      assert (x is None) == (y is None) and (x is None or (x == y).all()), (where, n)

  both(lambda e: e.sample_levels(np.arange(K) % 3 != 0))
  both(lambda e: e.pin_levels(np.arange(K, dtype=np.int32) % 5, np.arange(K) % 3 == 0))
  same('levels')
  both(lambda e: e.reset())
  same('reset')
  rs = np.random.RandomState(1)
  for t in range(18):
    acts = rs.randint(0, 17, K).astype(np.int32)
    ra, rb = both(lambda e: [x.copy() for x in e.step(acts, KINDS[t % 3])])
    assert all((x == y).all() for x, y in zip(ra, rb)), t
    same(t)
  assert (a.start_notes == 0).all() and a.stats[:, 0].sum() > 0


# ---- 3. a snapshot continues ------------------------------------------------------------------------------------
def test_a_snapshot_continues_with_the_same_starts():
  K, seed, length = 7, 33, 8
  table = np.array([11, 22, 33], np.int64)
  starts = [level_start({'wood': 3}, (33, 30), 'up'), level_start({'health': 3}, (31, 33), 'left'),
            np.zeros(START_WORDS, np.int32)]

  def make():
    env = SimtStartsEnv(num_envs=K, seed=seed, length=length, auto_reset=True)
    env.set_level_table(table, [1, 2, 3])
    env.set_level_starts(starts)
    return env

  a = make()
  a.sample_levels()
  a.reset()
  rs = np.random.RandomState(2)
  actions = rs.randint(0, 17, (40, K)).astype(np.int32)
  for t in range(13):
    a.step(actions[t], KINDS[t % 3])
  snap = {k: v.copy() for k, v in a.state.items()}
  notes, level = a.start_notes.copy(), a.level.copy()
  b = make()
  for k, v in snap.items():
    b.state[k][...] = v
  b.level[...] = level
  b.start_notes[...] = notes
  for t in range(13, 40):
    ra = [x.copy() for x in a.step(actions[t], KINDS[t % 3])]
    rb = [x.copy() for x in b.step(actions[t], KINDS[t % 3])]
    assert all((x == y).all() for x, y in zip(ra, rb)), t
  assert (b.start_notes == a.start_notes).all()
  for k, v in a.state.items():
    assert (v == b.state[k]).all(), k


# ---- 4. a goal with a start ----------------------------------------------------------------------------------------
def test_a_start_next_to_stone_with_a_wood_pickaxe_reaches_collect_stone():
  K, seed = 3, 8
  probe = SimtStartsEnv(num_envs=1, seed=0)
  W, H = probe.area
  mat, cre = np.full((W, H), GRASS, np.int64), np.zeros((W, H), np.int64)
  mat[10, 12] = STONE  # the start (10, 11) faces down onto it
  from tests.test_authored_levels import pack
  env = SimtStartsEnv(num_envs=K, seed=seed, length=50, auto_reset=True)
  env.set_level_table([1000, 2000])
  env.set_level_cache()
  env.fill()
  assert (env.author([0], pack([mat], [cre])) == 0).all()
  env.set_level_stats()
  env.set_level_goals([goal_mask('collect_stone'), 0])
  env.set_level_starts([level_start({'wood_pickaxe': 1}, (10, 11), 'down'), np.zeros(START_WORDS, np.int32)])
  env.pin_levels(np.array([0, 0, 1], np.int32))
  env.reset()
  assert env.state['pstate'][:2, PS['player_x']].tolist() == [10, 10]
  assert env.state['inventory'][:2, rules.ITEMS.index('wood_pickaxe')].tolist() == [1, 1]
  _, reward, done = env.step(np.full(K, rules.ACTIONS.index('do'), np.int32))
  assert reward[:2].tolist() == [1.0, 1.0] and done[:2].all() and not done[2], (reward, done)
  assert (env.state['final_stats'][:2, 23] == 2).all()
  assert env.stats[0, 0] == 2 and env.stats[0, 3] == 20
  assert (env.errors() == 0).all()


# ---- 5. host side, ABI, build ----------------------------------------------------------------------------------------
def test_level_start_and_host_validation():
  row = level_start()
  assert row.dtype == np.int32 and row.shape == (START_WORDS,)
  assert row.tolist() == [1, 32, 32, 3] + [9, 9, 9, 9] + [0] * 12
  row = level_start({'stone_pickaxe': 1, 'health': 4}, (3, 60), (1, 0), area=(64, 64))
  assert row[1:4].tolist() == [3, 60, 1] and row[4] == 4 and row[4 + rules.ITEMS.index('stone_pickaxe')] == 1
  assert level_start(pos=None, area=(37, 29))[1:3].tolist() == [18, 14]
  assert [int(level_start(facing=f)[3]) for f in ('left', 'right', 'up', 'down')] == [0, 1, 2, 3]
  for bad in (dict(inventory={'gold': 1}), dict(inventory={'wood': 10}), dict(inventory={'health': 0}),
              dict(inventory={'food': -1}), dict(pos=(64, 3)), dict(pos=(-1, 3)), dict(facing='north'),
              dict(facing=(1, 1)), dict(inventory={'wood': 1.5})):
    with pytest.raises(ValueError):
      level_start(**bad)

  class Fake:  # what set_level_starts reads before it touches a device
    _table, _table_len, _starts, _area = {'seeds': None}, 2, None, (64, 64)

  ok = level_start()
  for bad in ([ok], [ok, 'x'], [ok, dict(pos=(70, 0))], np.zeros((2, 19), np.int32), np.zeros((2, 20), np.float32),
              np.stack([ok, ok * 0 + 2]), torch.tensor(np.stack([ok, np.r_[1, 0, 0, 4, ok[4:]]])),
              np.stack([ok, np.r_[1, 0, 0, 0, 0, ok[5:]]])):
    with pytest.raises(ValueError):
      Env.set_level_starts(Fake(), bad)
  Fake._table = None
  with pytest.raises(RuntimeError, match='level table'):
    Env.set_level_starts(Fake(), [None, None])


def test_the_capacity_bounds_the_starts_and_removal_restores_the_reference():
  K, seed = 6, 9
  env = SimtStartsEnv(num_envs=K, seed=seed, length=50, auto_reset=True)
  env.set_level_table([1, 2, 3, 4], cap=4)
  rec = level_start({'wood': 2}, (33, 32), 'up')
  env.set_level_starts([rec] * 2, cap=2)  # entries 2 and 3 lie at or beyond the capacity
  env.pin_levels(np.arange(K, dtype=np.int32) % 4)
  env.reset()
  want = np.where((np.arange(K) % 4 < 2)[:, None], rec, 0)
  ep = env.episodes()
  for k in range(3):  # the running episode and the next two
    assert (env.start_notes[np.arange(K), (ep + k) & 3] == want).all(), env.start_notes
  with pytest.raises(RuntimeError, match='capacity'):
    env._check(env._L.hs_set_level_starts(env.h, env.starts.ctypes.data, env.start_notes.ctypes.data, 0))
  with pytest.raises(RuntimeError, match='notes'):
    env._check(env._L.hs_set_level_starts(env.h, env.starts.ctypes.data, None, 2))
  env.remove_level_starts()
  env.start_notes[:] = -7
  for _ in range(4):
    env.step(np.zeros(K, np.int32))
  assert (env.start_notes == -7).all()


def test_vector_env_passes_the_starts_through():
  calls = []

  class FakeEnv:

    def set_level_starts(self, starts):
      calls.append(('set', starts))

    @property
    def level_starts(self):
      calls.append(('read',))
      return 's'

  venv = vector.VectorEnv.__new__(vector.VectorEnv)
  venv.env = FakeEnv()
  venv.set_level_starts([None, None])
  assert venv.level_starts == 's'
  venv.set_level_starts(None)
  assert calls == [('set', [None, None]), ('read',), ('set', None)]


def test_abi_is_extended_not_changed():
  names = [f[0] for f in _cabi.CrState._fields_]
  assert len(names) == 24 and _cabi.ABI_VERSION == 6
  assert 'cr_set_level_starts' in _cabi.EXPORTS and 'cr_set_level_goals' in _cabi.EXPORTS
  header = (hostsim_env.HERE.parent / 'include' / 'crafter_b200.h').read_text()
  assert 'int cr_set_level_starts(cr_handle *h, const int32_t *starts, int32_t *notes, int cap);' in header
  assert '#define CR_START_WORDS 20' in header
  assert 'int cr_set_level_goals(cr_handle *h, const int32_t *goals, int32_t *notes, int cap);' in header
  assert ERR_LEVEL_START == 8


def test_the_tick_keeps_its_budget_and_the_start_kernels_do_not_spill(ptxas):  # noqa: F811
  for kernel in ('k_update', 'k_seed', 'k_install'):
    found = {targs: v for (name, targs), v in ptxas.items() if name == kernel}
    assert found and all(v.get('spill', 0) == 0 for v in found.values()), (kernel, found)
  update = [v for (name, _), v in ptxas.items() if name == 'k_update']
  assert all(v['regs'] == 58 for v in update), update
