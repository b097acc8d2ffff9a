"""Level goals (include/crafter_b200.h, cr_set_level_goals) on the product's kernels on the SIMT emulator
(tests/simt/simt_level_goals.cpp), against a twin batch without goals and a host restatement.

The restatement never reads the goal notes: it decides each episode's entry as tests/test_level_stats.py does
(`restated_draw` / `restated_entry` for a sampled env, the pinned entry below *n) and takes the goal of that entry from
the goal table as it stands when the entry is decided.  In every step it restates which episodes reached their goal
from the twin's achievements, and the twin then resets exactly those envs (`reset(mask)`), as a caller without goals
would.  So the goal run must equal the twin in every observation and in all of cr_state, except what the goal changes:
reward, done, ep_return, final_stats, PS_EP_LENGTH, the terminal outputs, final_world_seed / final_entry and the
statistics rows, which must equal the restatement.

1. A batch of level -1, fixed, sampled, pinned (one entry at or beyond *n), authored entries and two entries sharing a
   seed, some entries with goals a random policy reaches often (collect_sapling, collect_wood, wake_up, a conjunction):
   with and without auto_reset, all three kinds of step, the default and an odd geometry, with and without the cache;
   a mid-run goal rewrite reaches each env when the restatement says, and sample_levels / pin_levels make it hold
   from the next episode.
2. Goals registered with every entry 0 give a run identical to no goals, after every call.
3. A reached env stepped again without auto_reset reports done and pays nothing; the statistics count
   return_tenths == 10 * successes and terminated counts deaths only.
4. A snapshot of the state and the notes continues, in a fresh env, with the same goals.
5. goal_mask, host validation, the vector env's pass-through, the ABI, and the tick's register budget."""
import ctypes

import numpy as np
import pytest
import torch

from crafter_b200 import _cabi
from crafter_b200 import rules
from crafter_b200 import vector
from crafter_b200.env import Env, goal_mask
from tests import hostsim_env
from tests.test_authored_levels import ODD, oracle_packed
from tests.test_build_properties import ptxas  # noqa: F401  (fixture)
from tests.test_level_stats import Restated, SimtStatsEnv, simt_stats_lib
from tests.test_levels import KINDS, PS

FS_LENGTH, FS_DEAD, FS_INV, FS_POS = 22, 23, 24, 40
GOAL_BITS = (1 << 22) - 1
_LIB = []


def simt_goals_lib():
  """tests/simt/simt_level_goals.cpp: the statistics build plus hs_set_level_goals."""
  if not _LIB:
    here = hostsim_env.HERE
    src = here / 'simt' / 'simt_level_goals.cpp'
    out = here / 'simt' / '_build' / 'libsimt_level_goals.so'
    deps = [src] + [here / 'simt' / n for n in ('simt_level_stats.cpp', 'simt_authored.cpp', 'simt_level_cache.cpp',
                                                 'simt_level_sampler.cpp', 'simt_levels.cpp', 'simt_symbolic.cpp',
                                                 'simt_local.cpp', 'simt_env.cpp', 'simt.h')] + list(
        (here.parent / 'crafter_b200' / 'csrc').glob('*.h')) + [here.parent / 'include' / 'crafter_b200.h']
    hostsim_env._compile(out, src, deps)
    L = ctypes.CDLL(str(out))
    base = simt_stats_lib()
    for name in ('hs_create', 'hs_destroy', 'hs_reset', 'hs_step', 'hs_render', 'hs_semantic', 'hs_step_local',
                 'hs_local', 'hs_set_final_local', 'hs_step_symbolic', 'hs_symbolic', 'hs_set_final_symbolic',
                 'hs_set_level_buffers', 'hs_set_levels', 'hs_set_level_table', 'hs_sample_levels', 'hs_seed_only',
                 'hs_set_level_cache', 'hs_fill_level_cache', 'hs_author_levels', 'hs_pin_levels',
                 'hs_set_level_stats'):
      getattr(L, name).argtypes = getattr(base, name).argtypes
    L.hs_last_error.restype = ctypes.c_char_p
    L.hs_simt_blocks.restype = ctypes.c_long
    L.hs_set_level_goals.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_int]
    _LIB.append(L)
  return _LIB[0]


class SimtGoalsEnv(SimtStatsEnv):
  """SimtStatsEnv with the goal table and the goal notes in caller-owned numpy buffers."""

  goals = notes = None

  @staticmethod
  def _load(max_obj_tiles):
    assert max_obj_tiles is None
    return simt_goals_lib()

  def set_level_goals(self, goals, cap=None):
    """Register `goals` (padded with 0 to `cap`, None: the table's capacity) and notes filled with 0."""
    cap = cap or self.t_cap
    self.goals = np.zeros(cap, np.int32)
    self.goals[:len(goals)] = goals
    self.notes = np.zeros((self.B, 4), np.int32)
    self._check(self._L.hs_set_level_goals(self.h, self.goals.ctypes.data, self.notes.ctypes.data, cap))

  def remove_level_goals(self):
    self._check(self._L.hs_set_level_goals(self.h, None, None, 0))


# ---- the restatement ---------------------------------------------------------------------------------------------
class GoalRestated(Restated):
  """Restated (tests/test_level_stats.py) plus the goal of every decided episode, taken from `goals` (the goal run's
  table, rewritten in place by the tests) when its entry is decided."""

  def __init__(self, env, seed, cap, goals):
    super().__init__(env, seed, cap)
    self.goals = goals
    self.goal = [{} for _ in range(env.B)]

  def _decide(self, i, e):
    if e in self.decided[i]:
      return
    super()._decide(i, e)
    r = self.decided[i][e]
    self.goal[i][e] = int(self.goals[r]) & GOAL_BITS if 0 <= r < len(self.goals) else 0

  def goals_of(self, episodes):
    return np.array([self.goal[i].get(int(e), 0) for i, e in enumerate(episodes)], np.int64)

  def check_notes(self, where):
    ep = self.env.episodes()
    for i in range(self.env.B):
      for e in range(ep[i], ep[i] + 3):
        if e in self.goal[i]:
          assert self.env.notes[i, e & 3] == self.goal[i][e], (where, i, e, self.env.notes[i], self.goal[i])


# compared against the restatement instead; slot records below n_slots only: on a balance step the twin balances an
# env before its reset(mask), a goal run regenerates it without (its state is discarded), and the records beyond the
# new world's slots keep whatever the old world left there
STATE_EXCEPT = ('ep_return', 'final_stats', 'pstate', 'ents')
FINAL = ('final_obs', 'final_local', 'final_symbolic', 'final_semantic')


class Twin:
  """The goal run `a` (goals, statistics) and its twin `b` (no goals, statistics off), stepped side by side; `b`
  resets the envs the restatement says reached their goal.  Expectations of what the goal changes are kept here."""

  def __init__(self, K, seed, length, table, weights, goals, cached, auto_reset, stats_cap, **geometry):
    make = lambda: SimtGoalsEnv(num_envs=K, seed=seed, length=length, auto_reset=auto_reset, **geometry)
    self.a, self.b = make(), make()
    self.auto_reset = auto_reset
    for e in (self.a, self.b):
      e.set_level_table(table, weights, cap=len(table) + 2)
      if cached:
        e.set_level_cache()
        e.fill()
    self.a.set_level_stats(cap=stats_cap)
    self.a.set_level_goals(goals)
    self.res = GoalRestated(self.a, seed, stats_cap, self.a.goals)
    B = K
    self.paid = np.zeros(B)  # the goal run's return of the running episode of goal episodes
    self.fs = np.zeros((B, 42), np.int32)
    self.ep_length = np.zeros(B, np.int32)
    self.final_world_seed = np.zeros(B, np.int32)
    self.ret1 = np.zeros(B)
    self.last_done = np.zeros(B, bool)
    self.final = {n: None if getattr(self.a, n) is None else getattr(self.a, n).copy() for n in FINAL}
    self.reached_total = self.goal_episodes = 0

  def both(self, fn):
    return [fn(e) for e in (self.a, self.b)]

  def relevel(self, fn, mask):
    self.both(fn)
    self.res.relevel(mask)
    self.check('relevel')

  def reset(self, mask=None, kind='rgb'):
    oa, ob = self.both(lambda e: e.reset(mask, kind=kind).copy())
    self.res.started(mask)
    rows = slice(None) if mask is None else np.asarray(mask, bool)
    self.paid[rows] = 0
    assert (oa == ob).all()
    self.check('reset')

  def check(self, where):
    a, b = self.a, self.b
    for k, v in a.state.items():
      if k not in STATE_EXCEPT:
        assert (v == b.state[k]).all(), (where, k)
    cols = [c for c in range(16) if c != PS['episode_length']]
    assert (a.state['pstate'][:, cols] == b.state['pstate'][:, cols]).all(), where
    live = np.arange(a.state['ents'].shape[1]) < a.state['pstate'][:, PS['n_slots'], None]
    assert (a.state['ents'][live] == b.state['ents'][live]).all(), where
    assert (a.state['pstate'][:, PS['episode_length']] == self.ep_length).all(), where
    assert (a.state['final_stats'] == self.fs).all(), (where, np.argwhere(a.state['final_stats'] != self.fs)[:4])
    assert (a.final_world_seed == self.final_world_seed).all(), where
    has = self.res.goals_of(a.episodes()) != 0
    assert (a.state['ep_return'][:, 0] == np.where(has, self.paid, b.state['ep_return'][:, 0])).all(), where
    assert (a.state['ep_return'][:, 1] == self.ret1).all(), where
    assert (a.level == b.level).all(), where
    for n in FINAL:
      x = getattr(a, n)
      assert x is None or (x == self.final[n]).all(), (where, n)
    self.res.check_ring(where)
    self.res.check_notes(where)
    assert (a.stats == self.res.stats).all(), (where, np.argwhere(a.stats != self.res.stats)[:5])

  def step(self, t, actions, kind):
    a, b = self.a, self.b
    episode = a.episodes()
    before = b.state['pstate'][:, PS['unlocked']].astype(np.int64) & GOAL_BITS
    oa, ra, da = [x.copy() for x in a.step(actions, kind)]
    ob, rb, db = [x.copy() for x in b.step(actions, kind)]
    G = self.res.goals_of(episode)
    now = b.state['pstate'][:, PS['unlocked']].astype(np.int64) & GOAL_BITS
    if self.auto_reset:  # an env the twin ended has its next episode's state; its terminal record has the unlocks
      bits = (b.state['final_stats'][:, :22] >= 1).astype(np.int64) << np.arange(22)
      now = np.where(db, before | bits.sum(1), now)
    has = G != 0
    reached = has & ((now & G) == G)
    first = reached & ((before & G) != G)
    assert (ra == np.where(has, first.astype(np.float32), rb)).all(), (t, 'reward')
    assert (da == (db | reached)).all(), (t, 'done')
    self.reached_total += int(first.sum())
    self.goal_episodes += int((da & has).sum())
    self.paid += first
    # the terminal record of every env the goal run reports done, and its statistics
    for i in np.flatnonzero(da):
      if db[i]:
        row = b.state['final_stats'][i].copy()
      else:  # ended by its goal: the twin's state after the step, before its reset
        inv, ps = b.state['inventory'][i], b.state['pstate'][i]
        row = np.zeros(42, np.int32)
        row[:22], row[FS_LENGTH], row[FS_INV:FS_INV + 16] = b.state['achievements'][i], ps[PS['step']], inv
        row[FS_POS:FS_POS + 2] = ps[PS['player_x']], ps[PS['player_y']]
        row[FS_DEAD] = 1 if inv[0] <= 0 else 0
      row[FS_DEAD] |= 2 * int(reached[i])
      self.fs[i] = row
      self.ep_length[i] = row[FS_LENGTH]
      self.final_world_seed[i] = b.final_world_seed[i] if db[i] else b.state['pstate'][i, PS['world_seed']]
      self.ret1[i] = self.paid[i] if has[i] else b.state['ep_return'][i, 1]
      r = self.res.decided[i][episode[i]]
      self.res.final[i] = r
      if 0 <= r < self.res.cap:
        tenths = int(np.rint(10 * self.ret1[i]))
        self.res.stats[r, :5] += [1, row[FS_DEAD] & 1, row[FS_LENGTH], tenths, tenths * tenths]
        self.res.stats[r, 5:] += row[:22] >= 1
    assert (a.final_entry[da] == self.res.final[da]).all(), t
    # with auto_reset the twin resets what its goal ended; the terminal outputs of those envs are the twin's
    # before its reset
    if self.auto_reset:
      only = reached & ~db
      for n in FINAL:
        if self.final[n] is not None:
          self.final[n][db] = getattr(b, n)[db]
      if only.any() and (kind != 'rgb' or a.final_obs is not None):
        self.final[{'rgb': 'final_obs', 'semantic': 'final_local', 'symbolic': 'final_symbolic'}[kind]][only] = ob[only]
        if kind == 'semantic':  # the emulator's window step writes the terminal vectors too (tests/simt/simt_local.cpp)
          self.final['final_symbolic'][only] = b.observe('symbolic')[only]
        sem = self.final['final_semantic']
        sem[only] = b.semantic()[only].reshape(sem[only].shape)
      if only.any():
        ob = b.reset(only, kind=kind).copy()
      self.paid[da] = 0
      self.res.started(da)
    assert (oa == ob).all(), (t, 'obs', kind)
    self.last_done = da
    self.check(t)
    return da


GOAL_NAMES = ('collect_sapling', 'collect_wood', 'wake_up', ('collect_sapling', 'place_plant'))


@pytest.mark.parametrize('auto_reset', [True, False], ids=['auto_reset', 'no_auto_reset'])
@pytest.mark.parametrize('cached', [True, False], ids=['cached', 'uncached'])
@pytest.mark.parametrize('geometry', [dict(), ODD], ids=['default', 'odd_area'])
def test_the_goal_run_equals_its_twin_and_the_restatement(geometry, cached, auto_reset):
  K, seed, length = 14, 61, 40
  # entries 1 and 4 share a seed; entry 6 has weight 0 (pinned only); entry 5 lies at the statistics' capacity
  table = np.array([5, 1234567, 2 ** 31 - 2, 99, 1234567, 31337, 4242], np.int64)
  weights = [3, 2, 1, 2, 2, 1, 0]
  goals = [goal_mask(GOAL_NAMES[0]), goal_mask(GOAL_NAMES[1]), 0, goal_mask(GOAL_NAMES[2]), 0,
           goal_mask(GOAL_NAMES[3]), goal_mask(GOAL_NAMES[1])]
  tw = Twin(K, seed, length, table, weights, goals, cached, auto_reset, stats_cap=5, **geometry)
  if cached:  # authored entries: the generated worlds of other seeds under entries 2 and 6
    worlds = oracle_packed([77, 78], geometry)
    assert all((e.author([2, 6], worlds) == 0).all() for e in (tw.a, tw.b))
  kind = np.array([0, 1, 2, 3, 4, 4, 0, 1, 2, 3, 4, 4, 2, 4])  # 0: level -1, 1: fixed, 2 and 3: sampled, 4: pinned
  pins = np.zeros(K, np.int32)
  pins[kind == 4] = [6, 9, 5, 0, 3]  # entry 9 lies beyond *n = 7
  tw.relevel(lambda e: e.set_levels(1000 + np.arange(K), kind == 1), kind == 1)
  tw.relevel(lambda e: e.sample_levels((kind == 2) | (kind == 3)), (kind == 2) | (kind == 3))
  tw.relevel(lambda e: e.pin_levels(pins, kind == 4), kind == 4)
  tw.reset()
  rs = np.random.RandomState(seed)
  # actions that reach the goals often: collect (do), place a plant, walk
  policy = np.array([1, 2, 3, 4, 5, 5, 5, 5, 5, 5, 5, 10])
  stale = []
  for t in range(60):
    if t == 20:  # a goal rewrite: episodes decided from now on take the new goals, the two decided ones keep theirs
      tw.a.goals[1] = goal_mask('wake_up')
      tw.a.goals[0] = 0
      tw.check('rewrite')
      stale = [(i, e) for i in range(K) for e, g in tw.res.goal[i].items()
               if e > tw.a.episodes()[i] and tw.res.decided[i][e] in (0, 1)]
    if t == 30:  # sample_levels / pin_levels decide the next two episodes again: the new goals hold from the next one
      m = np.arange(K) == 2
      tw.relevel(lambda e: e.sample_levels(m), m)
      m = np.arange(K) == 3
      tw.relevel(lambda e: e.pin_levels(np.full(K, 1, np.int32), m), m)
      for i in (2, 3):
        e = tw.a.episodes()[i] + 1
        r = tw.res.decided[i][e]
        assert tw.res.goal[i][e] == (int(tw.a.goals[r]) if 0 <= r < 9 else 0)
    if not auto_reset and t % 15 == 14 and tw.last_done.any():  # the caller resets the done envs
      tw.reset(tw.last_done, kind=KINDS[t % 3])
    tw.step(t, policy[rs.randint(0, len(policy), K)].astype(np.int32), KINDS[t % 3])
  assert tw.reached_total >= 3, tw.reached_total
  assert tw.goal_episodes >= 3
  if auto_reset:
    assert stale, 'the rewrite found episodes decided before it'
  assert np.flatnonzero(tw.a.errors()).tolist() == [5]  # the env pinned to entry 9


def test_all_zero_goals_change_nothing():
  K, seed, length = 12, 5, 6
  table = np.array([7, 8, 9, 10], np.int64)

  def make(goals):
    env = SimtGoalsEnv(num_envs=K, seed=seed, length=length, auto_reset=True)
    env.set_level_table(table, [1, 2, 3, 1])
    env.set_level_cache()
    env.fill()
    env.set_level_stats()
    if goals:
      env.set_level_goals(np.zeros(4, np.int32))
    return env

  a, b = make(True), make(False)
  both = lambda fn: [fn(e) for e in (a, b)]

  def same(where):
    for k, v in a.state.items():
      assert (v == b.state[k]).all(), (where, k)
    for n in ('final_world_seed', 'final_entry', 'stats', 'ring', 'obs') + FINAL:
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
  assert (a.notes == 0).all() and a.stats[:, 0].sum() > 0


def test_a_reached_goal_pays_once_and_the_statistics_count_successes():
  K, seed = 6, 3
  env = SimtGoalsEnv(num_envs=K, seed=seed, length=200)
  env.set_level_table([10, 20, 30], cap=3)
  env.set_level_stats()
  env.set_level_goals([goal_mask('wake_up'), 0, goal_mask(['wake_up', 'collect_wood'])])
  env.pin_levels(np.arange(K, dtype=np.int32) % 3)
  env.reset()
  # sleep until woken up (energy starts full, so waking takes a while), then keep stepping
  paid = np.zeros(K)
  first_done = np.full(K, -1)
  for t in range(150):
    _, reward, done = env.step(np.full(K, 6, np.int32))
    paid += reward * (np.arange(K) % 3 != 1)
    newly = done & (first_done < 0)
    first_done[newly] = t
    after = (first_done >= 0) & (first_done < t) & (np.arange(K) % 3 == 0)
    if after.any():  # a goal env stepped again after reaching: done again, nothing paid
      assert done[after].all() and (reward[after] == 0).all(), t
  goal_envs = np.flatnonzero(np.arange(K) % 3 == 0)
  assert (first_done[goal_envs] >= 0).all(), first_done
  assert (paid[goal_envs] == 1).all(), paid
  assert (env.state['final_stats'][goal_envs, FS_DEAD] == 2).all()
  s = env.stats
  assert s[0, 3] == 10 * s[0, 0] and s[0, 1] == 0, s[0, :5]  # every counted episode succeeded; nobody died
  assert s[2, 3] == 0 and s[2, 0] == 0  # the conjunction is not reached by sleeping: no done, nothing counted


def test_a_snapshot_continues_with_the_same_goals():
  K, seed, length = 7, 33, 30
  table = np.array([11, 22, 33], np.int64)
  goals = [goal_mask('collect_sapling'), goal_mask('collect_wood'), 0]

  def make():
    env = SimtGoalsEnv(num_envs=K, seed=seed, length=length, auto_reset=True)
    env.set_level_table(table, [1, 2, 3])
    env.set_level_stats()
    env.set_level_goals(goals)
    return env

  a = make()
  a.sample_levels()
  a.reset()
  rs = np.random.RandomState(2)
  actions = rs.randint(0, 17, (60, K)).astype(np.int32)
  for t in range(25):
    a.step(actions[t], KINDS[t % 3])
  snap = {k: v.copy() for k, v in a.state.items()}
  notes, ring, final, level, at = a.notes.copy(), a.ring.copy(), a.final_entry.copy(), a.level.copy(), a.stats.copy()
  b = make()
  for k, v in snap.items():
    b.state[k][...] = v
  b.level[...] = level
  b.ring[...], b.final_entry[...], b.notes[...] = ring, final, notes
  for t in range(25, 60):
    ra = [x.copy() for x in a.step(actions[t], KINDS[t % 3])]
    rb = [x.copy() for x in b.step(actions[t], KINDS[t % 3])]
    assert all((x == y).all() for x, y in zip(ra, rb)), t
  assert (b.stats == a.stats - at).all() and (b.notes == a.notes).all()


# ---- 5. host side, ABI, build ----------------------------------------------------------------------------------------
def test_goal_mask_and_host_validation():
  A = rules.ACHIEVEMENTS
  assert goal_mask('collect_wood') == 1 << A.index('collect_wood')
  assert goal_mask(['wake_up', 'collect_sapling']) == (1 << A.index('wake_up')) | (1 << A.index('collect_sapling'))
  assert goal_mask(5) == 5 and goal_mask(()) == 0
  for bad in ('collect_gold', ['wake_up', 'fly'], 1 << 22, -1):
    with pytest.raises(ValueError):
      goal_mask(bad)

  class Fake:  # what set_level_goals reads before it touches a device
    _table, _table_len, _goals = {'seeds': None}, 3, None

  for bad in ([0, 1], ['wake_up', 'nope', 0], [0, 0, 1 << 22], np.array([0, -1, 0]), np.array([0.5, 0, 0]),
              torch.tensor([1 << 23, 0, 0])):
    with pytest.raises(ValueError):
      Env.set_level_goals(Fake(), bad)
  Fake._table = None
  with pytest.raises(RuntimeError, match='level table'):
    Env.set_level_goals(Fake(), [0, 0, 0])


def test_the_capacity_bounds_the_goals_and_removal_restores_the_reference():
  K, seed = 6, 9
  env = SimtGoalsEnv(num_envs=K, seed=seed, length=50, auto_reset=True)
  env.set_level_table([1, 2, 3, 4], cap=4)
  env.set_level_goals([goal_mask('wake_up')] * 2, cap=2)  # entries 2 and 3 lie at or beyond the capacity
  env.pin_levels(np.arange(K, dtype=np.int32) % 4)
  env.reset()
  want = np.where(np.arange(K) % 4 < 2, goal_mask('wake_up'), 0)
  ep = env.episodes()
  for k in range(3):  # the running episode and the next two
    assert (env.notes[np.arange(K), (ep + k) & 3] == want).all(), env.notes
  with pytest.raises(RuntimeError, match='capacity'):
    env._check(env._L.hs_set_level_goals(env.h, env.goals.ctypes.data, env.notes.ctypes.data, 0))
  env.remove_level_goals()
  env.notes[:] = -7
  for _ in range(4):
    env.step(np.zeros(K, np.int32))
  assert (env.notes == -7).all()


def test_vector_env_passes_the_goals_through():
  calls = []

  class FakeEnv:

    def set_level_goals(self, goals):
      calls.append(('set', goals))

    @property
    def level_goals(self):
      calls.append(('read',))
      return 'g'

  venv = vector.VectorEnv.__new__(vector.VectorEnv)
  venv.env = FakeEnv()
  venv.set_level_goals([1, 2])
  assert venv.level_goals == 'g'
  venv.set_level_goals(None)
  assert calls == [('set', [1, 2]), ('read',), ('set', None)]


def test_abi_is_extended_not_changed():
  names = [f[0] for f in _cabi.CrState._fields_]
  assert len(names) == 24 and _cabi.ABI_VERSION == 6
  assert 'cr_set_level_goals' in _cabi.EXPORTS and 'cr_set_level_stats' in _cabi.EXPORTS
  header = (hostsim_env.HERE.parent / 'include' / 'crafter_b200.h').read_text()
  assert 'int cr_set_level_goals(cr_handle *h, const int32_t *goals, int32_t *notes, int cap);' in header
  assert 'int cr_set_level_stats(cr_handle *h, int32_t *entry, int32_t *final_entry, int64_t *stats, int cap);' in header


def test_the_tick_keeps_its_budget_and_nothing_spills(ptxas):  # noqa: F811
  for kernel in ('k_update', 'k_seed'):
    found = {targs: v for (name, targs), v in ptxas.items() if name == kernel}
    assert found and all(v.get('spill', 0) == 0 for v in found.values()), (kernel, found)
  update = [v for (name, _), v in ptxas.items() if name == 'k_update']
  assert all(v['regs'] <= 60 for v in update), update
