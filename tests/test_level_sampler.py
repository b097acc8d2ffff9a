"""The level sampler (include/crafter_b200.h, cr_set_level_table / cr_sample_levels) on the product's kernels on the
SIMT emulator, and its draw with one lane (tests/hostsim/level_draw.cpp), against a restatement of the rule in
numpy and against the C oracle with levels (tests/oracle_levels.py).

* The draw restated: `restated_draw` below states the rule from oracle/keyed_rng.py's Philox and world_seed; the
  seeds k_seed decides, in its normal and its ahead pass, equal it for many tables, envs and episodes.
* The episodes are the oracle's: a batch that mixes level -1, fixed levels and sampled envs is compared with the
  oracle step by step over several auto-resets, all three kinds of step.
* Staleness is exactly as documented: the oracle side keeps, per env, the seeds that were decided and when.
* Edges, host validation, the ABI, the pass-through of the vector env, the distribution of the draws."""
import ctypes

import numpy as np
import pytest

from crafter_b200 import _cabi
from crafter_b200 import vector
from crafter_b200.env import MAX_LEVEL, MAX_WEIGHT_TOTAL, check_level_table, check_level_weights
from oracle import keyed_rng
from tests import hostsim_env
from tests.test_build_properties import ptxas  # noqa: F401  (fixture)
from tests.test_levels import KINDS, PS, OracleLevels, Run, SimtLevelsEnv, simt_levels_lib, world_seed

D_LEVEL = 6  # appended after keyed_rng.D_NOISE
SAMPLED = -2
ERR_LEVEL_TABLE = 4
NM_WORLD_SEED, NM_EPISODE, NM_VALID, NM_AHEAD_WORLD_SEED, NM_AHEAD_EPISODE, NM_AHEAD_VALID, NM_SEEDED = 1, 2, 3, 4, 5, 6, 7


# ---- the rule, restated ------------------------------------------------------------------------------
def restated_draw(j, episode, seeds, cum):
  """(world seed, empty) of episode `episode` of global env j from the table (seeds, inclusive cumulative weights)."""
  assert keyed_rng.D_NOISE + 1 == D_LEVEL
  key = world_seed(j, episode)
  total = int(cum[-1]) if len(cum) else 0
  if total == 0:
    return key, True
  w = keyed_rng.philox4x32((key, D_LEVEL), (0, 0, 0, 0))[0]
  t = (w * total) >> 32
  i = int(np.searchsorted(np.asarray(cum, np.uint64), np.uint64(t), side='right'))  # entries with cum <= t
  return int(seeds[i]), False


# ---- the builds --------------------------------------------------------------------------------------
_LIBS = {}


def simt_sampler_lib():
  """tests/simt/simt_level_sampler.cpp: the levels build plus hs_set_level_table, hs_sample_levels, hs_seed_only."""
  if 'simt' not in _LIBS:
    here = hostsim_env.HERE
    src = here / 'simt' / 'simt_level_sampler.cpp'
    out = here / 'simt' / '_build' / 'libsimt_level_sampler.so'
    deps = [src] + [here / 'simt' / n for n in ('simt_levels.cpp', 'simt_symbolic.cpp', 'simt_local.cpp', 'simt_env.cpp',
                                                 'simt.h')] + list(
        (here.parent / 'crafter_b200' / 'csrc').glob('*.h')) + [here.parent / 'include' / 'crafter_b200.h']
    hostsim_env._compile(out, src, deps)
    L = ctypes.CDLL(str(out))
    lev = simt_levels_lib()
    for name in ('hs_create', 'hs_destroy', 'hs_reset', 'hs_step', 'hs_render', 'hs_semantic', 'hs_recount',
                 'hs_step_local', 'hs_local', 'hs_set_final_local', 'hs_step_symbolic', 'hs_symbolic',
                 'hs_set_final_symbolic', 'hs_set_level_buffers', 'hs_set_levels'):
      getattr(L, name).argtypes = getattr(lev, name).argtypes
    L.hs_last_error.restype = ctypes.c_char_p
    L.hs_simt_blocks.restype = ctypes.c_long
    L.hs_set_level_table.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_int]
    L.hs_sample_levels.argtypes = [ctypes.c_void_p] * 2
    L.hs_seed_only.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
    _LIBS['simt'] = L
  return _LIBS['simt']


def one_lane_lib():
  if 'lane' not in _LIBS:
    here = hostsim_env.HERE
    src = here / 'hostsim' / 'level_draw.cpp'
    out = here / 'hostsim' / '_build' / 'liblevel_draw.so'
    hostsim_env._compile(out, src, [src] + list((here.parent / 'crafter_b200' / 'csrc').glob('*.h')))
    L = ctypes.CDLL(str(out))
    L.hs_level_draw.restype = ctypes.c_int64
    L.hs_level_draw.argtypes = [ctypes.c_int64, ctypes.c_int64, ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 3 + [
        ctypes.c_int]
    _LIBS['lane'] = L
  return _LIBS['lane']


class SimtSamplerEnv(SimtLevelsEnv):
  """SimtLevelsEnv with a level table in caller-owned numpy buffers, as a cr_set_level_table caller holds it."""

  @staticmethod
  def _load(max_obj_tiles):
    assert max_obj_tiles is None
    return simt_sampler_lib()

  def set_level_table(self, seeds, weights=None, cap=None):
    seeds = np.asarray(seeds, np.int64)
    n = len(seeds)
    cap = cap or max(n, 1)
    self.t_seeds, self.t_cum, self.t_n = np.zeros(cap, np.int32), np.zeros(cap, np.uint32), np.array([n], np.int32)
    self.t_seeds[:n] = seeds
    self.t_cap, self.registered = cap, True
    self.set_level_weights(np.ones(n, np.int64) if weights is None else weights)
    self._check(self._L.hs_set_level_table(self.h, self.t_seeds.ctypes.data, self.t_cum.ctypes.data, self.t_n.ctypes.data, cap))

  def set_level_weights(self, weights):
    """What Env.set_level_weights does: the cumulative sum in int64, stored as uint32 bit patterns."""
    w = np.asarray(weights, np.int64)
    self.t_cum[:len(w)] = (np.cumsum(w) & 0xFFFFFFFF).astype(np.uint32)

  def remove_level_table(self):
    self._check(self._L.hs_set_level_table(self.h, None, None, None, 0))
    self.registered = False

  def table(self):
    """(seeds, cum) the kernels see now."""
    if not getattr(self, 'registered', False):
      return np.zeros(0, np.int32), np.zeros(0, np.uint32)
    n = max(0, min(int(self.t_n[0]), self.t_cap))
    return self.t_seeds[:n], self.t_cum[:n]

  def sample_levels(self, mask=None):
    m = None if mask is None else np.ascontiguousarray(mask, np.uint8)
    self._check(self._L.hs_sample_levels(self.h, None if m is None else m.ctypes.data))

  def seed_only(self, count, ahead):
    self._L.hs_seed_only(self.h, count, ahead)

  def _check(self, rc):
    if rc != 0:
      raise RuntimeError(self._L.hs_last_error().decode())

  def errors(self):
    return self.state['pstate'][:, PS['error']].copy()

  def blocks(self):
    return int(self._L.hs_simt_blocks())


# ---- 1. the draw, restated ---------------------------------------------------------------------------------
def tables():
  rs = np.random.RandomState(11)
  seeds = lambda n: rs.randint(0, MAX_LEVEL + 1, n, dtype=np.int64)
  out = {
      'n1': (seeds(1), [7]),
      'n2': (seeds(2), [1, 3]),
      'n33': (seeds(33), rs.randint(1, 100, 33)),
      'n1000': (seeds(1000), rs.randint(0, 50, 1000)),
      'zeros_front_middle_end': (seeds(12), [0, 0, 5, 1, 0, 0, 0, 9, 2, 0, 0, 0]),
      'total_2_32_minus_1': (seeds(5), [2 ** 31, 2 ** 30, 2 ** 30 - 2, 0, 0]),
      'one_entry_holds_all': (seeds(40), [0] * 17 + [12345] + [0] * 22),
      'ends_of_the_seed_range': (np.array([0, MAX_LEVEL], np.int64), [1, 1]),
      'n2_20': (seeds(2 ** 20), rs.randint(0, 4000, 2 ** 20)),
  }
  w = out['total_2_32_minus_1'][1]
  w[-1] = MAX_WEIGHT_TOTAL - sum(w[:-1])
  assert sum(w) == MAX_WEIGHT_TOTAL and min(w) >= 0
  return out


TABLES = tables()


@pytest.mark.parametrize('name', list(TABLES))
def test_k_seed_draws_the_restated_seed_in_both_passes(name):
  """k_seed alone on a fresh handle of 37 envs (warps stride over the 3-SM grid) at a non-zero env_offset: the
  normal pass decides episode e + 1 of every env, the ahead pass the episode after it, for several e."""
  seeds, weights = TABLES[name]
  B, seed, offset = 37, 400, 1000
  env = SimtSamplerEnv(num_envs=B, seed=seed, env_offset=offset)
  env.set_level_table(seeds, weights)
  env.level[:] = SAMPLED
  s, cum = env.table()
  nm, ps = env.state['next_meta'], env.state['pstate']
  drawn = set()
  for e in (0, 1, 2, 7, 1000):
    ps[:, PS['episode']] = e
    nm[:, NM_SEEDED] = 0
    env.seed_only(B, 0)
    env.seed_only(B, 1)
    for i in range(B):
      want = [restated_draw(seed + offset + i, e + k, s, cum) for k in (1, 2)]
      assert not want[0][1] and (nm[i, NM_EPISODE], nm[i, NM_WORLD_SEED]) == (e + 1, want[0][0]), (name, e, i, 'normal')
      assert (nm[i, NM_AHEAD_EPISODE], nm[i, NM_AHEAD_WORLD_SEED]) == (e + 2, want[1][0]), (name, e, i, 'ahead')
      drawn |= {want[0][0], want[1][0]}
    assert nm[:, NM_SEEDED].all() and nm[:, NM_AHEAD_VALID].all()
  assert not env.errors().any()
  positive = set(np.asarray(seeds)[np.asarray(weights) > 0].tolist())
  assert drawn <= positive, 'an entry of weight 0 was drawn'
  if len(positive) > 1:
    assert len(drawn) > 1


@pytest.mark.parametrize('name', list(TABLES))
def test_one_lane_bisection_draws_the_restated_seed(name):
  seeds, weights = TABLES[name]
  L = one_lane_lib()
  s = np.asarray(seeds, np.int32)
  cum = (np.cumsum(np.asarray(weights, np.int64)) & 0xFFFFFFFF).astype(np.uint32)
  n = np.array([len(s)], np.int32)
  for env in range(0, 300, 7):
    for episode in (1, 2, 50):
      got = L.hs_level_draw(9, 64, env, episode, s.ctypes.data, cum.ctypes.data, n.ctypes.data, len(s))
      assert got == restated_draw(9 + 64 + env, episode, s, cum)[0], (name, env, episode)
  # n beyond the capacity is read as the capacity; no table, n = 0 and a zero total are "empty"
  big = np.array([len(s) + 5], np.int32)
  assert L.hs_level_draw(9, 0, 3, 1, s.ctypes.data, cum.ctypes.data, big.ctypes.data, len(s)) == restated_draw(12, 1, s, cum)[0]
  zero = np.zeros(1, np.int32)
  key = world_seed(12, 1)
  assert L.hs_level_draw(9, 0, 3, 1, s.ctypes.data, cum.ctypes.data, zero.ctypes.data, len(s)) == -1 - key
  assert L.hs_level_draw(9, 0, 3, 1, None, None, None, 0) == -1 - key
  none = np.zeros(len(s), np.uint32)
  assert L.hs_level_draw(9, 0, 3, 1, s.ctypes.data, none.ctypes.data, n.ctypes.data, len(s)) == -1 - key


# ---- 5. distribution ---------------------------------------------------------------------------------
def test_draws_follow_the_weights():
  """Weights 1 : 2 : 5 over three seeds, 64 envs x 60 episodes of k_seed on the emulator: chi-square at a fixed seed."""
  from scipy import stats
  B, seed = 64, 2024
  env = SimtSamplerEnv(num_envs=B, seed=seed)
  table = np.array([111, 222, 333], np.int64)
  env.set_level_table(table, [1, 2, 5])
  env.level[:] = SAMPLED
  nm, ps = env.state['next_meta'], env.state['pstate']
  counts = np.zeros(3, np.int64)
  for e in range(0, 60, 2):
    ps[:, PS['episode']] = e
    nm[:, NM_SEEDED] = 0
    env.seed_only(B, 0)
    env.seed_only(B, 1)
    for col in (NM_WORLD_SEED, NM_AHEAD_WORLD_SEED):
      counts += (nm[:, col][:, None] == table[None, :]).sum(0)
  total = B * 60
  assert counts.sum() == total
  p = stats.chisquare(counts, total * np.array([1, 2, 5]) / 8).pvalue
  assert p > 0.001, (counts, p)


# ---- the oracle side of a run with sampled envs ----------------------------------------------------------
class OracleSampled(OracleLevels):
  """OracleLevels whose sampled envs start each episode on the seed that was DECIDED for it: a seed is decided from
  the table as it stands when the env becomes sampled (its next two episodes) and when an episode starts (every
  episode up to the one after next that has no seed yet) -- the normal and the ahead pass of k_seed."""

  def __init__(self, K, seed, env, **kwargs):
    super().__init__(K, seed, **kwargs)
    self.env, self.seed = env, seed
    self.sampled = np.zeros(K, bool)
    self.decided = [{} for _ in range(K)]
    self.empty = np.zeros(K, bool)  # envs that must carry ERR_LEVEL_TABLE
    self.history = [[] for _ in range(K)]  # (episode, world seed) of the episodes started on a drawn seed

  @property
  def level(self):
    return np.where(self.sampled, SAMPLED, OracleLevels.level.fget(self))

  def _decide(self, i, episode):
    if episode not in self.decided[i]:
      ws, empty = restated_draw(self.seed + i, episode, *self.env.table())
      self.decided[i][episode] = ws
      self.empty[i] |= empty

  def sample(self, mask=None):
    for i, ref in enumerate(self.refs):
      if mask is None or mask[i]:
        self.sampled[i], self.decided[i] = True, {}
        self._decide(i, ref.episode + 1)
        self._decide(i, ref.episode + 2)

  def set_levels(self, levels, mask=None):
    super().set_levels(levels, mask)
    for i in range(len(self.refs)):
      if mask is None or mask[i]:
        self.sampled[i], self.decided[i] = False, {}

  def reset(self, i):
    ref = self.refs[i]
    if self.sampled[i]:
      e = ref.episode + 1
      for k in (e, e + 1, e + 2):
        self._decide(i, k)
      ref.set_level(self.decided[i][e])
      self.history[i].append((e, self.decided[i][e]))
    return ref.reset()


class SampledRun(Run):
  """tests/test_levels.Run with the sampler: SimtSamplerEnv beside OracleSampled."""

  def __init__(self, K=4, seed=30, length=4, start_step=None, **geometry):
    self.env = SimtSamplerEnv(num_envs=K, seed=seed, length=length, auto_reset=True, **geometry)
    self.ora = OracleSampled(K, seed, self.env, length=length, **geometry)
    self.K, self.grid, self.start_step = K, self.env.grid, start_step
    self.reached = dict(episodes=0, terminal=0, night=0, kinds=set(), seeds=set())
    self.rs = np.random.RandomState(seed)

  def sample_levels(self, mask=None):
    self.env.sample_levels(mask)
    self.ora.sample(mask)
    assert self.env.counters() == (0, 0), 'work-list counters not zero after cr_sample_levels'

  def check_errors(self):
    want = np.where(self.ora.empty, ERR_LEVEL_TABLE, 0)
    assert (self.env.errors() == want).all(), (self.env.errors(), want)


# ---- 2. episodes are the oracle's ---------------------------------------------------------------------
def test_mixed_sampled_and_fixed_levels_over_several_episodes():
  """13 envs: level -1, fixed seeds and sampled envs (table with a zero-weight entry), sampling chosen before the
  first reset for some and mid-run for others; frame, window and vector steps in turn across several auto-resets.
  final_world_seed names the sampled world, which replays through reset(mask, levels)."""
  K, seed, length = 13, 50, 4
  run = SampledRun(K=K, seed=seed, length=length)
  table = np.array([5, 1234567, MAX_LEVEL, 0, 99, 31337], np.int64)
  run.env.set_level_table(table, [3, 1, 2, 0, 2, 1], cap=16)
  early = np.zeros(K, bool)
  early[[1, 2, 5, 8, 9, 12]] = True
  run.sample_levels(early)  # before the first reset
  levels = np.full(K, -1, np.int32)
  levels[[3, 4, 7]] = [42, 1234567, MAX_LEVEL]
  fixed = ~early
  run.set_levels(levels, fixed)
  run.reset()
  late = np.zeros(K, bool)
  late[[0, 4]] = True
  log = []  # (final world seed, actions, rewards, terminal semantic map) of sampled episodes
  acts, rewards = [[] for _ in range(K)], [[] for _ in range(K)]
  for t in range(18):
    if t == 5:
      run.sample_levels(late)  # mid-episode: from each env's next episode on
    if t == 11:
      run.set_levels(np.full(K, 77, np.int32), np.arange(K) == 9)  # out of sampling again
    actions = run.rs.randint(0, 17, K).astype(np.int32)
    done = run.step(t, KINDS[t % 3], actions)
    for i in range(K):
      acts[i].append(int(actions[i]))
      rewards[i].append(float(run.env.reward[i]))
      if done[i]:
        if run.ora.sampled[i] and len(run.ora.history[i]) >= 2:  # the episode that ended started on a drawn seed
          log.append((int(run.env.final_world_seed[i]), acts[i], rewards[i], run.env.final_semantic[i].copy()))
        acts[i], rewards[i] = [], []
  run.check_errors()
  assert not run.ora.empty.any()
  assert run.reached['kinds'] == set(KINDS) and run.reached['episodes'] >= 3 * K
  drawn = {ws for h in run.ora.history for _, ws in h}
  assert len(drawn) >= 4 and 0 not in drawn and drawn <= set(table.tolist()), drawn
  assert (run.env.level[early & (np.arange(K) != 9)] == SAMPLED).all() and run.env.level[9] == 77
  assert 77 in run.reached['seeds']
  # replay a logged sampled episode on another batch as a level
  ws, actions, want_rewards, want_semantic = log[-1]
  assert ws in table
  replay = SimtLevelsEnv(num_envs=2, seed=999, length=length, auto_reset=True)
  replay.reset(levels=np.array([-1, ws], np.int32))
  for k, act in enumerate(actions):
    _, reward, done = replay.step(np.array([0, act], np.int32))
    assert float(reward[1]) == want_rewards[k] and bool(done[1]) == (k == len(actions) - 1), k
  assert replay.final_world_seed[1] == ws and (replay.final_semantic[1] == want_semantic).all()


@pytest.mark.parametrize('order', ['m', 'o'])
def test_sampling_does_not_depend_on_where_the_ahead_pass_runs(order, monkeypatch):
  """The ahead seed runs beside the terrain on the device: after k_wg_mat or after k_wg_obj must do as well."""
  monkeypatch.setenv('CR_SIMT_WG_ORDER', order)
  run = SampledRun(K=5, seed=8, length=3)
  run.env.set_level_table([10, 20, 30, 40], [1, 1, 1, 1])
  run.sample_levels()
  run.reset()
  for t in range(9):
    run.step(t, KINDS[t % 3])
  run.check_errors()


# ---- 3. staleness ------------------------------------------------------------------------------------
def test_weight_updates_reach_an_env_after_at_most_two_episodes():
  K, seed, length = 6, 77, 3
  run = SampledRun(K=K, seed=seed, length=length)
  table = np.array([101, 202, 303, 404, 505], np.int64)
  hot = 404
  run.env.set_level_table(table)
  run.sample_levels()
  run.reset()
  for t in range(4):
    run.step(t, 'rgb')
  # a weight update generates no world and launches nothing
  before = {k: run.env.state[k].copy() for k in ('next_mat', 'next_ents', 'next_meta', 'perm')}
  blocks = run.env.blocks()
  run.env.set_level_weights([0, 0, 0, 9, 0])
  assert run.env.blocks() == blocks
  assert all((run.env.state[k] == v).all() for k, v in before.items())
  started = [len(h) for h in run.ora.history]
  # envs 0 and 1 ask for the new table now: their next worlds are drawn and generated again, once
  again = np.arange(K) < 2
  run.sample_levels(again)
  assert run.env.counters() == (0, 0)
  nm = run.env.state['next_meta']
  for i in range(K):
    if again[i]:
      assert nm[i, NM_VALID] == 1 and nm[i, NM_WORLD_SEED] == hot and nm[i, NM_AHEAD_WORLD_SEED] == hot
    else:
      assert (nm[i] == before['next_meta'][i]).all() and (run.env.state['next_mat'][i] == before['next_mat'][i]).all()
  for t in range(4, 4 + 4 * length):
    run.step(t, KINDS[t % 3])
  run.check_errors()
  stale = 0
  for i in range(K):
    new = [ws for _, ws in run.ora.history[i][started[i]:]]  # the episodes started after the update
    assert len(new) >= 4, new
    if again[i]:
      assert all(ws == hot for ws in new), (i, new)
    else:
      assert all(ws == hot for ws in new[2:]), (i, new)  # from its third new episode at the latest
      # its first two were drawn from the old table (uniform over five seeds): played as drawn
      want = [restated_draw(seed + i, e, table, np.arange(1, 6))[0] for e, _ in run.ora.history[i][started[i]:started[i] + 2]]
      assert new[:2] == want, (i, new, want)
      stale += sum(ws != hot for ws in new[:2])
  assert stale > 0, 'no stale seed was played: the test did not see the staleness'


# ---- 4. edges ----------------------------------------------------------------------------------------
def test_an_empty_table_plays_the_reference_sequence_and_raises_the_error_bit():
  K, seed = 4, 21
  run = SampledRun(K=K, seed=seed, length=3)
  run.env.set_level_table([1, 2, 3], [1, 1, 1], cap=8)
  run.env.t_n[0] = 0  # envs 0, 1: sampled from an empty table
  run.sample_levels(np.array([1, 1, 0, 0], bool))
  run.env.t_n[0] = 3
  run.env.set_level_weights([0, 0, 0])  # env 2: a zero total
  run.sample_levels(np.array([0, 0, 1, 0], bool))
  run.env.set_level_weights([1, 0, 0])
  run.reset()
  assert run.env.world_seed().tolist() == [world_seed(seed + i, 1) for i in range(K)]
  assert run.env.errors().tolist() == [4, 4, 4, 0]
  for t in range(7):
    run.step(t, KINDS[t % 3])
  # the two seeds decided from the empty table were played as decided, the later ones come from the table
  for i in range(3):
    assert [ws for _, ws in run.ora.history[i]][:3] == [world_seed(seed + i, 1), world_seed(seed + i, 2), 1]
  run.check_errors()  # sticky, and env 3 never raised it
  assert run.env.level.tolist() == [SAMPLED] * 3 + [-1]


def test_removing_the_table_and_shrinking_n_are_harmless():
  K, seed = 3, 9
  run = SampledRun(K=K, seed=seed, length=3)
  run.env.set_level_table(np.arange(100, 140), cap=64)
  run.sample_levels()
  run.reset()
  for t in range(4):
    run.step(t, 'semantic')
  assert {ws for h in run.ora.history for _, ws in h} <= set(range(100, 140))
  run.env.t_n[0] = 2  # below the index of seeds already drawn and waiting in next_meta
  run.env.set_level_weights([1, 1])
  for t in range(4, 12):
    run.step(t, 'semantic')
  assert all(h[-1][1] in (100, 101) for h in run.ora.history)
  assert not run.env.errors().any()
  run.env.remove_level_table()  # envs still sampled: as the empty table
  with pytest.raises(RuntimeError, match='no level table'):
    run.env.sample_levels()
  for t in range(12, 24):
    run.step(t, 'symbolic')
  for i, h in enumerate(run.ora.history):
    assert h[-1] == (h[-1][0], world_seed(seed + i, h[-1][0]))
  run.check_errors()
  assert (run.env.errors() == ERR_LEVEL_TABLE).all()
  # set_levels takes the envs out of sampling
  run.set_levels(np.array([-1, 55, -1], np.int32))
  for t in range(24, 30):
    run.step(t, 'rgb')
  assert run.env.level.tolist() == [-1, 55, -1] and 55 in run.reached['seeds']


def test_sample_levels_needs_a_table_and_the_level_buffer():
  env = SimtSamplerEnv(num_envs=2, seed=3)
  with pytest.raises(RuntimeError, match='no level table'):
    env.sample_levels()
  with pytest.raises(RuntimeError, match='seeds without'):
    env._check(env._L.hs_set_level_table(env.h, env.level.ctypes.data, None, None, 4))
  bare = SimtSamplerEnv(num_envs=2, seed=3, level_buffers=False)
  bare.set_level_table([1, 2])
  with pytest.raises(RuntimeError, match='no level buffer'):
    bare.sample_levels()
  assert env.counters() == (0, 0) and bare.counters() == (0, 0)
  bare.reset()
  assert bare.world_seed().tolist() == [world_seed(3, 1), world_seed(4, 1)]


def test_the_table_is_checked_on_the_host():
  import torch
  seeds, weights = check_level_table([3, 0, MAX_LEVEL])
  assert seeds.tolist() == [3, 0, MAX_LEVEL] and weights.tolist() == [1, 1, 1] and weights.dtype == torch.int64
  seeds, weights = check_level_table(np.array([1, 2], np.uint32), torch.tensor([0, MAX_WEIGHT_TOTAL]))
  assert weights.tolist() == [0, MAX_WEIGHT_TOTAL]
  for bad in ([-1, 2], [0, MAX_LEVEL + 1], np.array([2 ** 32 - 1], np.uint32)):
    with pytest.raises(ValueError, match='world seeds|out of range'):
      check_level_table(bad)
  with pytest.raises(ValueError, match='at least one'):
    check_level_table(np.zeros(0, np.int64))
  with pytest.raises(ValueError, match='shape'):
    check_level_table(np.zeros((2, 2), np.int64))
  with pytest.raises(ValueError, match='shape'):
    check_level_table([1, 2, 3], [1, 1])
  for dtype in (np.float32, bool):
    with pytest.raises(ValueError, match='integers'):
      check_level_table(np.zeros(3, dtype))
    with pytest.raises(ValueError, match='integers'):
      check_level_table([1, 2, 3], np.ones(3, dtype))
  with pytest.raises(ValueError, match='integers'):
    check_level_weights(torch.ones(3), 3)
  with pytest.raises(ValueError, match=r'integers in \[0'):
    check_level_table([1, 2], [1, -1])
  with pytest.raises(ValueError, match='total weight'):
    check_level_table([1, 2], [0, 0])
  with pytest.raises(ValueError, match='total weight'):
    check_level_table([1, 2], [MAX_WEIGHT_TOTAL, 1])
  assert check_level_weights(np.array([0, 7], np.int16), 2).tolist() == [0, 7]


def test_vector_env_passes_the_sampler_through():
  calls = []

  class FakeEnv:

    def set_level_table(self, seeds, weights=None):
      calls.append(('table', seeds, weights))

    def set_level_weights(self, weights):
      calls.append(('weights', weights))

    def sample_levels(self, mask=None):
      calls.append(('sample', mask))

  venv = vector.VectorEnv.__new__(vector.VectorEnv)
  venv.env = FakeEnv()
  venv.set_level_table([1, 2])
  venv.set_level_table([1, 2], [3, 4])
  venv.set_level_weights([5, 6])
  venv.sample_levels()
  venv.sample_levels([1, 0])
  assert calls == [('table', [1, 2], None), ('table', [1, 2], [3, 4]), ('weights', [5, 6]), ('sample', None),
                   ('sample', [1, 0])]


def test_abi_is_extended_not_changed():
  names = [f[0] for f in _cabi.CrState._fields_]
  assert names[-2:] == ['level', 'final_world_seed'] and len(names) == 24 and _cabi.ABI_VERSION == 6
  assert {'cr_set_level_table', 'cr_sample_levels'} <= set(_cabi.EXPORTS)
  header = (hostsim_env.HERE.parent / 'include' / 'crafter_b200.h').read_text()
  assert '#define CR_ABI_VERSION 6' in header and 'int cr_sample_levels(' in header and 'int cr_set_level_table(' in header


def test_seed_and_sample_kernels_do_not_spill(ptxas):  # noqa: F811
  for kernel in ('k_seed', 'k_sample_levels'):
    found = {targs: v for (name, targs), v in ptxas.items() if name == kernel}
    assert len(found) == 1 and all(v.get('spill', 0) == 0 for v in found.values()), (kernel, found)
