"""Per-level episode statistics (include/crafter_b200.h, cr_set_level_stats) on the product's kernels on the SIMT
emulator (tests/simt/simt_level_stats.cpp), against a numpy restatement.

The restatement never reads the entry notes: it decides each episode's entry itself, when the contract says its seed
is decided (when an env is put on a level, table or entry: its next two episodes; when an episode starts: every
episode up to the one after next that has none yet), from the env's level as it stands then -- a sampled env's entry
is the index `restated_draw` (tests/test_level_sampler.py) draws for (j, e) from the table as it stands, a pinned env's
is its entry below *n -- and counts every step's done envs from that step's done, final_stats and ep_return.

1. A batch of level -1, fixed, sampled, pinned (one entry at or beyond *n) and authored entries, with a table in
   which two entries share a seed, counts what the restatement counts, across auto-resets and all three kinds of
   step, at the default and an odd geometry; mid-episode set_levels, sample_levels, pin_levels and weight rewrites
   attribute as documented, and entries at or beyond the statistics' capacity are not counted.
2. Every output and all of cr_state equal, after every call, those of the same batch with no ring, and with a ring
   but no statistics; with or without the level cache.
3. Without auto_reset a repeated done counts once per step; reset() of a running episode counts nothing; removal.
4. A snapshot of the state and the notes taken mid-episode continues, in a fresh env, with the same counts.
5. level_scores, the ABI, the vector env's pass-through, and no spills."""
import ctypes

import numpy as np
import pytest
import torch

from crafter_b200 import _cabi
from crafter_b200 import rules
from crafter_b200 import vector
from crafter_b200.env import LEVEL_STATS, LEVEL_STATS_COLUMNS, level_scores
from oracle import keyed_rng
from tests import hostsim_env
from tests.test_authored_levels import ODD, SimtAuthoredEnv, oracle_packed, simt_authored_lib
from tests.test_build_properties import ptxas  # noqa: F401  (fixture)
from tests.test_level_sampler import D_LEVEL, restated_draw
from tests.test_levels import KINDS, PS, world_seed

FS_LENGTH, FS_DEAD = 22, 23
_LIB = []


def simt_stats_lib():
  """tests/simt/simt_level_stats.cpp: the authored build plus hs_set_level_stats."""
  if not _LIB:
    here = hostsim_env.HERE
    src = here / 'simt' / 'simt_level_stats.cpp'
    out = here / 'simt' / '_build' / 'libsimt_level_stats.so'
    deps = [src] + [here / 'simt' / n for n in ('simt_authored.cpp', 'simt_level_cache.cpp', 'simt_level_sampler.cpp',
                                                 'simt_levels.cpp', 'simt_symbolic.cpp', 'simt_local.cpp', 'simt_env.cpp',
                                                 'simt.h')] + list(
        (here.parent / 'crafter_b200' / 'csrc').glob('*.h')) + [here.parent / 'include' / 'crafter_b200.h']
    hostsim_env._compile(out, src, deps)
    L = ctypes.CDLL(str(out))
    base = simt_authored_lib()
    for name in ('hs_create', 'hs_destroy', 'hs_reset', 'hs_step', 'hs_render', 'hs_semantic', 'hs_step_local',
                 'hs_local', 'hs_set_final_local', 'hs_step_symbolic', 'hs_symbolic', 'hs_set_final_symbolic',
                 'hs_set_level_buffers', 'hs_set_levels', 'hs_set_level_table', 'hs_sample_levels', 'hs_seed_only',
                 'hs_set_level_cache', 'hs_fill_level_cache', 'hs_author_levels', 'hs_pin_levels'):
      getattr(L, name).argtypes = getattr(base, name).argtypes
    L.hs_last_error.restype = ctypes.c_char_p
    L.hs_simt_blocks.restype = ctypes.c_long
    L.hs_set_level_stats.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_int]
    _LIB.append(L)
  return _LIB[0]


class SimtStatsEnv(SimtAuthoredEnv):
  """SimtAuthoredEnv with the entry notes, final_entry and the statistics rows in caller-owned numpy buffers."""

  ring = final_entry = stats = None

  @staticmethod
  def _load(max_obj_tiles):
    assert max_obj_tiles is None
    return simt_stats_lib()

  def set_level_stats(self, stats=True, cap=None):
    """Register a ring (filled with -1), final_entry and, with `stats`, `cap` rows (None: the table's capacity)."""
    self.ring = np.full((self.B, 4), -1, np.int32)
    self.final_entry = np.full(self.B, -1, np.int32)
    cap = cap or self.t_cap
    self.stats = np.zeros((cap, LEVEL_STATS_COLUMNS), np.int64) if stats else None
    self._check(self._L.hs_set_level_stats(self.h, self.ring.ctypes.data, self.final_entry.ctypes.data,
                                           None if self.stats is None else self.stats.ctypes.data, cap if stats else 0))

  def remove_level_stats(self):
    self._check(self._L.hs_set_level_stats(self.h, None, None, None, 0))

  def episodes(self):
    return self.state['pstate'][:, PS['episode']].copy()


# ---- the restatement ---------------------------------------------------------------------------------------------
def restated_entry(j, episode, seeds, cum):
  """The table entry the draw of (global env j, episode) picks, -1 for an empty table: the index behind
  restated_draw's seed."""
  ws, empty = restated_draw(j, episode, seeds, cum)
  if empty:
    return -1
  w = keyed_rng.philox4x32((world_seed(j, episode), D_LEVEL), (0, 0, 0, 0))[0]
  i = int(np.searchsorted(np.asarray(cum, np.uint64), np.uint64((w * int(cum[-1])) >> 32), side='right'))
  assert int(seeds[i]) == ws
  return i


class Restated:
  """The entries and the statistics of a SimtStatsEnv's batch, restated from the contract (see the module docstring).
  The env is read for its level buffer, table, episode counters and per-step outputs only, never for its notes."""

  def __init__(self, env, seed, cap):
    self.env, self.seed, self.cap = env, seed, cap
    self.decided = [{} for _ in range(env.B)]
    self.stats = np.zeros((cap, LEVEL_STATS_COLUMNS), np.int64)
    self.final = np.full(env.B, -1, np.int64)

  def _decide(self, i, e):
    if e in self.decided[i]:
      return
    level = int(self.env.level[i])
    seeds, cum = self.env.table()
    if level == -2:
      r = restated_entry(self.seed + i, e, seeds, cum)
    elif level <= -3:
      r = -3 - level if -3 - level < len(seeds) else -1
    else:
      r = -1
    self.decided[i][e] = r

  def relevel(self, mask=None):
    """After set_levels / sample_levels / pin_levels: the next two episodes of the masked envs are decided again."""
    ep = self.env.episodes()
    for i in range(self.env.B):
      if mask is None or mask[i]:
        self.decided[i] = {k: v for k, v in self.decided[i].items() if k <= ep[i]}
        self._decide(i, ep[i] + 1)
        self._decide(i, ep[i] + 2)

  def started(self, mask=None):
    """After episodes started (reset, or auto-reset in a step)."""
    ep = self.env.episodes()
    for i in range(self.env.B):
      if mask is None or mask[i]:
        for k in range(3):
          self._decide(i, ep[i] + k)

  def count(self, done, episode_before):
    fs, ret = self.env.state['final_stats'], self.env.state['ep_return']
    for i in np.flatnonzero(done):
      r = self.decided[i][episode_before[i]]
      self.final[i] = r
      if 0 <= r < self.cap:
        tenths = int(np.rint(10 * ret[i, 1]))
        row = self.stats[r]
        row[:5] += [1, fs[i, FS_DEAD], fs[i, FS_LENGTH], tenths, tenths * tenths]
        row[5:] += fs[i, :22] >= 1

  def check_ring(self, where):
    """The notes the kernels wrote for the running episode and the next two equal the decided entries."""
    ep = self.env.episodes()
    for i in range(self.env.B):
      for e in range(ep[i], ep[i] + 3):
        if e in self.decided[i]:
          assert self.env.ring[i, e & 3] == self.decided[i][e], (where, i, e, self.env.ring[i], self.decided[i])


# ---- 1 and 2: a mixed batch ------------------------------------------------------------------------------------------
class Trio:
  """The same batch three times -- `full` with the ring and the statistics, `ring` with the ring only, `bare` with
  neither -- compared after every call; `full`'s statistics against the restatement."""

  def __init__(self, K, seed, length, table, weights, cached, stats_cap, **geometry):
    make = lambda: SimtStatsEnv(num_envs=K, seed=seed, length=length, auto_reset=True, **geometry)
    self.full, self.ring, self.bare = make(), make(), make()
    self.envs = (self.full, self.ring, self.bare)
    for e in self.envs:
      e.set_level_table(table, weights, cap=len(table) + 2)
    for e in (self.full, self.ring, self.bare)[:3 if cached == 'all' else 1]:
      e.set_level_cache()
      e.fill()
    self.full.set_level_stats(cap=stats_cap)
    self.ring.set_level_stats(stats=False)
    self.res = Restated(self.full, seed, stats_cap)

  def all(self, fn):
    return [fn(e) for e in self.envs]

  def check(self, where):
    a = self.full
    for b in self.envs[1:]:
      for k, v in a.state.items():
        assert (v == b.state[k]).all(), (where, k)
      for name in ('final_world_seed', 'level', 'final_semantic', 'final_local', 'final_symbolic', 'final_obs', 'obs'):
        x, y = getattr(a, name), getattr(b, name)
        assert (x is None) == (y is None) and (x is None or (x == y).all()), (where, name)
    assert (self.ring.ring == self.full.ring).all() and (self.ring.final_entry == self.full.final_entry).all(), where
    self.res.check_ring(where)
    assert (self.full.stats == self.res.stats).all(), (where, np.argwhere(self.full.stats != self.res.stats)[:5])

  def relevel(self, fn, mask):
    self.all(fn)
    self.res.relevel(mask)
    self.check('relevel')

  def step(self, t, actions, kind):
    before = self.full.episodes()
    outs = self.all(lambda e: [x.copy() for x in e.step(actions, kind)])
    for o in outs[1:]:
      for x, y in zip(outs[0], o):
        assert (x == y).all(), t
    done = outs[0][2].astype(bool)
    self.res.count(done, before)
    assert (self.full.final_entry[done] == self.res.final[done]).all(), t
    self.res.started(done)
    self.check(t)
    return done


@pytest.mark.parametrize('cached', ['all', 'full_only'], ids=['cached', 'cache_only_in_the_counting_env'])
@pytest.mark.parametrize('geometry', [dict(), ODD], ids=['default', 'odd_area'])
def test_stats_equal_the_restatement_and_change_no_output(geometry, cached):
  K, seed, length = 14, 61, 3
  # entries 1 and 4 share a seed; entry 6 has weight 0 (pinned only); entry 5 lies at the statistics' capacity
  table = np.array([5, 1234567, 2 ** 31 - 2, 99, 1234567, 31337, 4242], np.int64)
  weights = [3, 2, 1, 2, 2, 1, 0]
  trio = Trio(K, seed, length, table, weights, cached, stats_cap=5, **geometry)
  if cached == 'all':  # authored entries: the generated worlds of other seeds under entries 2 and 6
    worlds = oracle_packed([77, 78], geometry)
    for e in trio.envs:
      assert (e.author([2, 6], worlds) == 0).all()
  kind = np.array([0, 1, 2, 3, 4, 4, 0, 1, 2, 3, 4, 4, 2, 4])  # 0: level -1, 1: fixed, 2 and 3: sampled, 4: pinned
  pins = np.zeros(K, np.int32)
  pins[kind == 4] = [6, 9, 5, 2, 0]  # entry 9 lies beyond *n = 7
  trio.relevel(lambda e: e.set_levels(1000 + np.arange(K), kind == 1), kind == 1)
  trio.relevel(lambda e: e.sample_levels((kind == 2) | (kind == 3)), (kind == 2) | (kind == 3))
  trio.relevel(lambda e: e.pin_levels(pins, kind == 4), kind == 4)
  trio.all(lambda e: e.reset())
  trio.res.started()
  trio.check('reset')
  rs = np.random.RandomState(seed)
  done_total = 0
  for t in range(16):
    if t == 4:  # mid-episode: sampled envs onto a fixed level and a pinned entry, a fixed one into sampling
      m = np.arange(K) == 2
      trio.relevel(lambda e: e.set_levels(np.full(K, 555, np.int32), m), m)
      m = np.arange(K) == 3
      trio.relevel(lambda e: e.pin_levels(np.full(K, 4, np.int32), m), m)
      m = np.arange(K) == 1
      trio.relevel(lambda e: e.sample_levels(m), m)
    if t == 7:  # a weight rewrite: seeds decided from now on are drawn from the new weights
      trio.all(lambda e: e.set_level_weights([0, 1, 0, 0, 5, 0, 0]))
      trio.check('weights')
    if t == 10:
      m = np.arange(K) == 7
      trio.relevel(lambda e: e.sample_levels(m), m)
    done_total += trio.step(t, rs.randint(0, 17, K).astype(np.int32), KINDS[t % 3]).sum()
  s = trio.full.stats
  decided = {r for d in trio.res.decided for r in d.values()}
  assert {-1, 1, 2, 4, 5, 6} <= decided, decided
  assert done_total >= 3 * K and s[:, 0].sum() >= K, (done_total, s[:, 0])
  assert s[1, 0] > 0 and s[4, 0] > 0, 'the two entries of one seed are counted apart'
  assert np.flatnonzero(trio.full.errors()).tolist() == [5]  # the env pinned to entry 9


# ---- 3. without auto_reset; reset; removal -----------------------------------------------------------------------
def test_repeated_done_counts_per_step_and_reset_counts_nothing():
  K, seed = 4, 8
  env = SimtStatsEnv(num_envs=K, seed=seed, length=3)
  env.set_level_table([10, 20])
  env.set_level_stats()
  res = Restated(env, seed, 2)
  env.pin_levels(np.array([0, 1, 0, 1], np.int32))
  res.relevel()
  env.reset()
  res.started()
  for t in range(5):  # done at step 3, then twice more
    before = env.episodes()
    _, _, done = env.step(np.zeros(K, np.int32))
    res.count(done, before)
    assert (env.stats == res.stats).all(), t
  assert env.stats[:, 0].tolist() == [2 * 3, 2 * 3], env.stats[:, 0]
  assert env.stats[0, 2] == 2 * (3 + 4 + 5)
  env.reset(np.array([1, 1, 0, 0], bool))  # ends done episodes and nothing is counted
  res.started(np.array([1, 1, 0, 0], bool))
  before_stats = env.stats.copy()
  env.step(np.zeros(K, np.int32))
  env.reset(np.array([1, 0, 0, 0], bool))  # a running episode
  res.started(np.array([1, 0, 0, 0], bool))
  assert (env.stats[:, 0] == before_stats[:, 0] + [1, 1]).all()  # envs 2 and 3 were still done; 0 and 1 run
  res.relevel(np.zeros(K, bool))
  res.check_ring('reset')
  # removal: nothing is written any more
  env.remove_level_stats()
  frozen = env.stats.copy()
  env.final_entry[:] = -9
  for _ in range(4):
    env.step(np.zeros(K, np.int32))
  assert (env.stats == frozen).all() and (env.final_entry == -9).all()


def test_entries_at_or_beyond_cap_are_ignored_and_notes_are_kept_without_stats():
  K, seed = 6, 19
  env = SimtStatsEnv(num_envs=K, seed=seed, length=2, auto_reset=True)
  env.set_level_table([1, 2, 3, 4], cap=4)
  env.set_level_stats(cap=2)
  env.pin_levels(np.arange(K, dtype=np.int32) % 4)
  env.reset()
  for _ in range(6):
    _, _, done = env.step(np.zeros(K, np.int32))
  assert env.stats[:, 0].tolist() == [2 * 3, 2 * 3] and env.final_entry.tolist() == [0, 1, 2, 3, 0, 1]
  notes_only = SimtStatsEnv(num_envs=K, seed=seed, length=2, auto_reset=True)
  notes_only.set_level_table([1, 2, 3, 4], cap=4)
  notes_only.set_level_stats(stats=False)
  notes_only.pin_levels(np.arange(K, dtype=np.int32) % 4)
  notes_only.reset()
  for _ in range(6):
    notes_only.step(np.zeros(K, np.int32))
  assert (notes_only.ring == env.ring).all() and (notes_only.final_entry == env.final_entry).all()
  with pytest.raises(RuntimeError, match='capacity'):
    env._check(env._L.hs_set_level_stats(env.h, env.ring.ctypes.data, None, env.stats.ctypes.data, 0))


# ---- 4. a snapshot continues with the same counts ------------------------------------------------------------------
def test_a_snapshot_taken_mid_episode_continues_with_the_same_counts():
  K, seed, length = 7, 33, 4
  table = np.array([11, 22, 33], np.int64)

  def make():
    env = SimtStatsEnv(num_envs=K, seed=seed, length=length, auto_reset=True)
    env.set_level_table(table, [1, 2, 3])
    env.set_level_stats()
    return env

  a = make()
  a.sample_levels()
  a.pin_levels(np.full(K, 2, np.int32), np.arange(K) % 3 == 0)
  a.reset()
  rs = np.random.RandomState(2)
  actions = rs.randint(0, 17, (20, K)).astype(np.int32)
  for t in range(9):
    a.step(actions[t], KINDS[t % 3])
  snap = {k: v.copy() for k, v in a.state.items()}
  notes, final, level, at = a.ring.copy(), a.final_entry.copy(), a.level.copy(), a.stats.copy()
  assert (a.state['pstate'][:, PS['step']] > 0).any()
  b = make()
  for k, v in snap.items():
    b.state[k][...] = v
  b.level[...] = level
  b.ring[...], b.final_entry[...] = notes, final
  for t in range(9, 20):
    ra = [x.copy() for x in a.step(actions[t], KINDS[t % 3])]
    rb = [x.copy() for x in b.step(actions[t], KINDS[t % 3])]
    assert all((x == y).all() for x, y in zip(ra, rb)), t
  assert (b.stats == a.stats - at).all() and b.stats[:, 0].sum() >= K


# ---- 5. host side, ABI, build ----------------------------------------------------------------------------------------
def test_level_scores_follow_the_reference_formula():
  rs = np.random.RandomState(0)
  episodes = np.array([10, 0, 3, 1], np.int64)
  ach = np.minimum(rs.randint(0, 11, (4, 22)), episodes[:, None])
  stats = {k: torch.zeros(4, dtype=torch.int64) for k in LEVEL_STATS}
  stats['episodes'] = torch.from_numpy(episodes)
  stats['achievements'] = torch.from_numpy(ach)
  percent, score = level_scores(stats)
  assert percent.shape == (4, 22) and score.shape == (4,)
  with np.errstate(invalid='ignore', divide='ignore'):
    want = 100 * ach / episodes[:, None]
  want_score = np.exp(np.mean(np.log(1 + want), -1)) - 1  # analysis/common.py:47-55
  ok = episodes > 0
  assert np.allclose(percent.numpy()[ok], want[ok], rtol=0, atol=1e-12)
  assert np.allclose(score.numpy()[ok], want_score[ok], rtol=1e-12)
  assert torch.isnan(percent[1]).all() and torch.isnan(score[1])
  full = {k: torch.zeros(1, dtype=torch.int64) for k in LEVEL_STATS}
  full['episodes'][0] = 4
  full['achievements'] = torch.full((1, 22), 4, dtype=torch.int64)
  assert abs(float(level_scores(full)[1][0]) - 100) < 1e-9
  assert LEVEL_STATS_COLUMNS == 5 + len(rules.ACHIEVEMENTS) == 27


def test_vector_env_passes_the_statistics_through():
  calls = []

  class FakeEnv:

    def set_level_stats(self, enabled=True):
      calls.append(('set', enabled))

    def level_stats(self):
      calls.append(('read',))
      return 's'

    def clear_level_stats(self, entries=None):
      calls.append(('clear', entries))

  venv = vector.VectorEnv.__new__(vector.VectorEnv)
  venv.env = FakeEnv()
  venv.set_level_stats()
  assert venv.level_stats() == 's'
  venv.clear_level_stats([3])
  venv.set_level_stats(False)
  assert calls == [('set', True), ('read',), ('clear', [3]), ('set', False)]


def test_abi_is_extended_not_changed():
  names = [f[0] for f in _cabi.CrState._fields_]
  assert len(names) == 24 and _cabi.ABI_VERSION == 6
  assert 'cr_set_level_stats' in _cabi.EXPORTS
  header = (hostsim_env.HERE.parent / 'include' / 'crafter_b200.h').read_text()
  assert 'int cr_set_level_stats(cr_handle *h, int32_t *entry, int32_t *final_entry, int64_t *stats, int cap);' in header
  assert 'int cr_set_level_cache(cr_handle *h, uint8_t *mat, void *ents, int32_t *meta, int32_t *tag, int32_t *row, int cap);' in header


def test_counting_kernels_do_not_spill_and_the_tick_keeps_its_budget(ptxas):  # noqa: F811
  for kernel in ('k_update', 'k_seed'):
    found = {targs: v for (name, targs), v in ptxas.items() if name == kernel}
    assert found and all(v.get('spill', 0) == 0 for v in found.values()), (kernel, found)
  update = [v for (name, _), v in ptxas.items() if name == 'k_update']
  assert all(v['regs'] <= 60 for v in update), update  # the tick's count before the statistics
