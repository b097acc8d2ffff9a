"""Levels (include/crafter_b200.h, cr_set_levels) on the product's kernels on the SIMT emulator, against the C
oracle with levels (tests/oracle_levels.py): which world seed each env's episodes play, sticky across auto-resets, changed
only from an env's next episode on, with `info['final_world_seed']` naming the world of an episode that ended.

* The golden fixtures tie levels to the unmodified reference: episode k of fixture env i played world seed
  world_seed(seed0 + i, k); a batch with another seed, the episode put on another env index, replays that
  episode's recorded digests from its actions.
* A mixed batch of 13 envs (the emulator's 3-SM grids stride) rotates frame, window and vector steps on one
  handle across several episodes, at the default geometry and three others.
* Changes of level mid-episode, twice before an episode ends, back to -1, before the first reset, and with
  reset(mask, levels).
* A logged episode replays on another batch from its final_world_seed and its actions."""
import ctypes
import zlib

import numpy as np
import pytest

from crafter_b200 import _cabi
from crafter_b200 import state as state_lib
from crafter_b200.env import MAX_LEVEL, check_levels
from crafter_b200 import vector
from oracle import canon
from tests import hostsim_env
from tests import oracle_levels
from tests import parity
from tests import geometry_cases as gc
from tests.golden_util import Fixture
from tests.test_build_properties import ptxas  # noqa: F401  (fixture)
from tests.test_schedule_knobs import SLEEP
from tests.test_semantic_obs import grid_of, oracle_window, window_problem
from tests.test_symbolic_obs import oracle_vector, vector_problem

PS = state_lib.PS
KINDS = ('rgb', 'semantic', 'symbolic')

# ---- the emulator build ----------------------------------------------------------------------------
_LEVELS_LIB = []


def simt_levels_lib():
  """tests/simt/simt_levels.cpp: the symbolic build (frame, window and vector steps) plus hs_set_levels and
  hs_set_level_buffers."""
  if not _LEVELS_LIB:
    from tests.test_symbolic_obs import simt_symbolic_lib
    here = hostsim_env.HERE
    src = here / 'simt' / 'simt_levels.cpp'
    out = here / 'simt' / '_build' / 'libsimt_levels.so'
    deps = [src] + [here / 'simt' / n for n in ('simt_symbolic.cpp', 'simt_local.cpp', 'simt_env.cpp', 'simt.h')] + list(
        (here.parent / 'crafter_b200' / 'csrc').glob('*.h')) + [here.parent / 'include' / 'crafter_b200.h']
    hostsim_env._compile(out, src, deps)
    L = ctypes.CDLL(str(out))
    sym = simt_symbolic_lib()  # the argument types of the entry points simt_levels.cpp includes
    for name in ('hs_create', 'hs_destroy', 'hs_reset', 'hs_step', 'hs_render', 'hs_semantic', 'hs_recount',
                 'hs_step_local', 'hs_local', 'hs_set_final_local', 'hs_step_symbolic', 'hs_symbolic',
                 'hs_set_final_symbolic'):
      getattr(L, name).argtypes = getattr(sym, name).argtypes
    L.hs_last_error.restype = ctypes.c_char_p
    L.hs_set_level_buffers.argtypes = [ctypes.c_void_p] * 3
    L.hs_set_levels.argtypes = [ctypes.c_void_p] * 3
    _LEVELS_LIB.append(L)
  return _LEVELS_LIB[0]


class SimtLevelsEnv(hostsim_env.SimtEnv):
  """One emulator handle with levels (cr_state.level, final_world_seed) that steps frames (cr_step), windows
  (cr_step_local) or vectors (cr_step_symbolic), chosen per call, with the terminal output of every kind on
  (terminal frames where the geometry takes them).  `level_buffers=False`: cr_state.level stays NULL."""

  def __init__(self, num_envs, level_buffers=True, **kwargs):
    geometry = {k: kwargs[k] for k in ('area', 'view', 'size') if k in kwargs}
    frames_ok = bool(hostsim_env.geom(**geometry)['terminal_ok'])
    super().__init__(num_envs=num_envs, final_obs=frames_ok and kwargs.get('auto_reset', False), **kwargs)
    B = num_envs
    self.grid = grid_of(kwargs.get('view', (9, 9)))
    dim = 22 * self.grid[0] * self.grid[1] + 22
    self.local = np.zeros((B,) + self.grid, np.uint8)
    self.vec = np.zeros((B, dim), np.float32)
    self.final_local = np.zeros((B,) + self.grid, np.uint8)
    self.final_symbolic = np.zeros((B, dim), np.float32)
    if self.final_semantic is None:
      self.final_semantic = np.zeros((B,) + self.area, np.uint8)
    self._L.hs_set_final_local(self.h, self.final_local.ctypes.data, self.final_semantic.ctypes.data)
    self._L.hs_set_final_symbolic(self.h, self.final_symbolic.ctypes.data, self.final_semantic.ctypes.data)
    self.level = np.full(B, -1, np.int32)
    self.final_world_seed = np.zeros(B, np.int32)
    if level_buffers:
      self._L.hs_set_level_buffers(self.h, self.level.ctypes.data, self.final_world_seed.ctypes.data)

  @staticmethod
  def _load(max_obj_tiles):
    assert max_obj_tiles is None
    return simt_levels_lib()

  def set_levels(self, levels, mask=None):
    """cr_set_levels (hs_set_levels); raises RuntimeError with its message when it fails."""
    lv = np.ascontiguousarray(levels, np.int32)
    m = None if mask is None else np.ascontiguousarray(mask, np.uint8)
    if self._L.hs_set_levels(self.h, None if m is None else m.ctypes.data, lv.ctypes.data) != 0:
      raise RuntimeError(self._L.hs_last_error().decode())

  def reset(self, mask=None, levels=None, kind='rgb'):
    if levels is not None:
      self.set_levels(levels, mask)
    m = None if mask is None else np.ascontiguousarray(mask, np.uint8)
    self._L.hs_reset(self.h, None if m is None else m.ctypes.data, self.obs.ctypes.data if kind == 'rgb' else None)
    return self.observe(kind)

  def observe(self, kind):
    """The observation of `kind` as the state stands (the frames only after a frame step / reset)."""
    if kind == 'semantic':
      self._L.hs_local(self.h, self.local.ctypes.data)
      return self.local
    if kind == 'symbolic':
      self._L.hs_symbolic(self.h, self.vec.ctypes.data)
      return self.vec
    return self.obs

  def step(self, actions, kind='rgb'):
    a = np.ascontiguousarray(actions, np.int32)
    fn = {'rgb': self._L.hs_step, 'semantic': self._L.hs_step_local, 'symbolic': self._L.hs_step_symbolic}[kind]
    out = {'rgb': self.obs, 'semantic': self.local, 'symbolic': self.vec}[kind]
    fn(self.h, a.ctypes.data, out.ctypes.data, self.reward.ctypes.data, self.done.ctypes.data)
    return out, self.reward, self.done.astype(bool)

  def final(self, kind):
    return {'rgb': self.final_obs, 'semantic': self.final_local, 'symbolic': self.final_symbolic}[kind]

  def world_seed(self):
    """info['world_seed']."""
    return self.state['pstate'][:, PS['world_seed']].copy()

  def counters(self):
    return int(self.state['reset_count'][0]), int(self.state['balance_count'][0])


# ---- the oracle side ---------------------------------------------------------------------------------
class OracleLevels:
  """K oracle envs with levels (tests/oracle_levels.LevelEnv; env i: seed + i), and the world seed each one plays,
  restated from the definition: the level when it is >= 0, else world_seed(seed + i, episode)."""

  def __init__(self, K, seed, **kwargs):
    self.refs = [oracle_levels.LevelEnv(seed=seed + i, **kwargs) for i in range(K)]

  @property
  def level(self):
    return np.array([r.level for r in self.refs], np.int64)

  @property
  def ws(self):
    return np.array([r.world_seed for r in self.refs], np.int64)

  def set_levels(self, levels, mask=None):
    for i, ref in enumerate(self.refs):
      if mask is None or mask[i]:
        ref.set_level(int(levels[i]))

  def reset(self, i):
    return self.refs[i].reset()

  def jump(self, i, step):
    """Move env i's step counter (nightfall inside short runs), keeping its world."""
    ref = self.refs[i]
    ref.import_state(ref.export_state(), int(step), ref.episode, ref.world_seed)


def expected_obs(ref, kind, frame, grid):
  if kind == 'semantic':
    return oracle_window(ref, grid)[1]
  if kind == 'symbolic':
    return oracle_vector(ref, grid)[1]
  return frame


def obs_problem(kind, got, want, grid):
  if kind == 'semantic':
    return window_problem(got, want)
  if kind == 'symbolic':
    return vector_problem(got, want, grid)
  return parity.frame_problem(got, want)


class Run:
  """A SimtLevelsEnv with auto_reset beside OracleLevels, compared after every call: reward, done, canonical
  state, info['world_seed'], the levels, and the obs of the step kind; for the envs that finished the terminal
  obs of the step kind, the terminal semantic map and info['final_world_seed']."""

  def __init__(self, K=4, seed=30, length=4, start_step=None, **geometry):
    self.env = SimtLevelsEnv(num_envs=K, seed=seed, length=length, auto_reset=True, **geometry)
    self.ora = OracleLevels(K, seed, length=length, **geometry)
    self.K, self.grid, self.start_step = K, self.env.grid, start_step
    self.reached = dict(episodes=0, terminal=0, night=0, kinds=set(), seeds=set())
    self.rs = np.random.RandomState(seed)

  def _jump(self, ids):
    if self.start_step is None:
      return
    for i in ids:
      self.env.state['pstate'][i, PS['step']] = self.start_step
      self.ora.jump(i, self.start_step)

  def set_levels(self, levels, mask=None):
    self.env.set_levels(levels, mask)
    self.ora.set_levels(levels, mask)
    assert self.env.counters() == (0, 0), 'work-list counters not zero after cr_set_levels'

  def reset(self, mask=None, levels=None, kind='rgb'):
    if levels is not None:
      self.ora.set_levels(levels, mask)
    obs = self.env.reset(mask, levels, kind).copy()
    assert self.env.counters() == (0, 0), 'work-list counters not zero after cr_reset'
    ids = range(self.K) if mask is None else np.flatnonzero(mask)
    for i in ids:
      frame = self.ora.reset(i)
      want = expected_obs(self.ora.refs[i], kind, frame, self.grid)
      problem = obs_problem(kind, obs[i], want, self.grid)
      assert problem is None, ('reset', kind, i, problem)
    self._jump(ids)
    self._check_state('reset')
    return obs

  def _check_state(self, where):
    assert (self.env.level == self.ora.level).all(), (where, 'levels', self.env.level, self.ora.level)
    ws = self.env.world_seed()
    for i, ref in enumerate(self.ora.refs):
      assert ws[i] == self.ora.ws[i], (where, i, 'world_seed', int(ws[i]), int(self.ora.ws[i]))
      problem = canon.diff(ref.export_state(), self.env.snapshot(i))
      assert problem is None, (where, i, problem)

  def step(self, t, kind, actions=None):
    if actions is None:
      actions = self.rs.randint(0, 17, self.K).astype(np.int32)
      actions[self.rs.rand(self.K) < 0.2] = SLEEP
    obs, reward, done = self.env.step(actions, kind)
    obs = obs.copy()
    self.reached['kinds'].add(kind)
    finished = []
    for i, ref in enumerate(self.ora.refs):
      where = (t, kind, i)
      frame, r, d = ref.step(int(actions[i])) if kind == 'rgb' else (None,) + ref.step_norender(int(actions[i]))
      assert np.float32(r) == reward[i] and d == bool(done[i]), where + ('reward / done',)
      if d:
        final = self.env.final(kind)
        if final is not None:
          want = expected_obs(ref, kind, frame, self.grid)
          problem = obs_problem(kind, final[i], want, self.grid)
          assert problem is None, where + ('terminal obs', problem)
          self.reached['terminal'] += 1
        assert (self.env.final_semantic[i] == ref.semantic()).all(), where + ('terminal semantic',)
        assert self.env.final_world_seed[i] == self.ora.ws[i], where + (
            'final_world_seed', int(self.env.final_world_seed[i]), int(self.ora.ws[i]))
        self.reached['seeds'].add(int(self.ora.ws[i]))
        frame = self.ora.reset(i)
        self.reached['episodes'] += 1
        finished.append(i)
      want = expected_obs(ref, kind, frame, self.grid)  # the first of the next episode where one ended
      problem = obs_problem(kind, obs[i], want, self.grid)
      assert problem is None, where + ('obs', problem)
      if ref.export_state()['daylight'] < 0.5:
        self.reached['night'] += 1
    self._jump(finished)
    self._check_state((t, kind))
    return done


def world_seed(seed, episode):
  from oracle import oracle_env
  return oracle_env.world_seed(seed, episode)


# ---- 1. tied to the unmodified reference ------------------------------------------------------------
# (fixture, fixture env, episode): episodes after the first, which the default sequence of a fresh env never reaches
FIXTURE_EPISODES = [('default_short', 1, 2), ('default_short', 0, 4), ('default_fighter', 2, 3), ('tiny_area', 3, 2),
                    ('default_random', 5, 1)]


@pytest.mark.parametrize('name,i,k', FIXTURE_EPISODES)
def test_level_replays_a_recorded_reference_episode(name, i, k):
  """Episode k of fixture env i played world seed world_seed(seed0 + i, k) on the reference.  A fresh batch with
  another seed plays it on another env index as a level and must reproduce the recorded reset and step digests,
  reward, done and frame CRCs from that episode's actions (inventory boost applied after the reset as recorded)."""
  fx = Fixture(name)
  done_at = np.flatnonzero(fx.env(i, 'done'))
  first = 0 if k == 1 else int(done_at[k - 2]) + 1
  last = int(done_at[k - 1]) if k - 1 < len(done_at) else fx.T - 1
  B, j = 3, 2 if i != 2 else 1
  env = SimtLevelsEnv(num_envs=B, seed=fx.seed0 + 1000, **fx.kwargs)
  levels = np.full(B, -1, np.int32)
  levels[j] = world_seed(fx.seed0 + i, k)
  obs = env.reset(levels=levels)
  assert env.world_seed()[j] == levels[j]
  if fx.boost:
    env.set_inventory(fx.boost, env_ids=[j])
    obs = env.render()
  st = env.snapshot(j)
  for key, v in canon.digest(st).items():
    assert v == fx.env(i, f'reset_{key}_crc')[k - 1], (name, i, k, 'reset', key)
  assert zlib.crc32(np.ascontiguousarray(obs[j]).tobytes()) == fx.env(i, 'reset_obs_crc')[k - 1], 'reset obs'
  actions = np.zeros(B, np.int32)
  for t in range(first, last + 1):
    actions[j] = fx.env(i, 'actions')[t]
    obs, reward, done = env.step(actions)
    where = (name, i, k, t)
    assert bool(done[j]) == bool(fx.env(i, 'done')[t]), where + ('done',)
    assert reward[j] == np.float32(fx.env(i, 'reward')[t]), where + ('reward',)
    st = env.snapshot(j)
    for key, v in canon.digest(st).items():
      assert v == fx.env(i, f'{key}_crc')[t], where + (key,)
    assert zlib.crc32(np.ascontiguousarray(obs[j]).tobytes()) == fx.env(i, 'obs_crc')[t], where + ('obs',)
  assert last - first + 1 > 0


# ---- 2. a mixed batch over several episodes ----------------------------------------------------------
K_MIXED = 13
MIXED = {  # name: (geometry, length, start step after every reset or None)
    'default': (gc.kwargs('default'), 4, None),
    'odd_geometry_night': (gc.kwargs('odd_geometry'), 160, 155),
    'view5x7': (gc.kwargs('view5x7'), 5, None),
    'tiny_area_night': (gc.kwargs('tiny_area'), 160, 156),
}


def mixed_levels(seed):
  """-1, the two ends of the range, one seed shared by four envs, and one env on another env's default world."""
  shared = 1234567
  lv = [-1, 0, MAX_LEVEL, shared, shared, -1, world_seed(seed + 0, 2), shared, 42, -1, shared, 7, 2 ** 30]
  assert len(lv) == K_MIXED
  return np.array(lv, np.int32)


@pytest.mark.parametrize('name', list(MIXED))
def test_mixed_levels_over_several_episodes(name):
  geometry, length, start = MIXED[name]
  seed = 50
  run = Run(K=K_MIXED, seed=seed, length=length, start_step=start, **geometry)
  run.reset(levels=mixed_levels(seed))
  steps = 15
  for t in range(steps):
    run.step(t, KINDS[t % 3])
  r = run.reached
  assert r['kinds'] == set(KINDS)
  assert r['episodes'] >= 2 * K_MIXED, r
  assert {0, MAX_LEVEL, 1234567} <= r['seeds'], r['seeds']
  if start is not None:
    assert r['night'] > 0, r


# ---- 3. changing levels ----------------------------------------------------------------------------------
def test_level_changes_take_effect_from_the_next_episode():
  """set_levels mid-episode (the running episode is left alone), two assignments before an episode ends (the last
  wins), back to -1 (the reference sequence at the env's next episode number), for at least three episodes after
  each call so that a stale ahead seed shows; the frame, window and vector steps in turn."""
  K, seed = 5, 61
  run = Run(K=K, seed=seed, length=4)
  run.reset()
  lv = lambda *v: np.array(v, np.int32)
  schedule = {
      1: (lv(111, 222, 333, -1, -1), None),                            # mid-episode, every env
      2: (lv(0, 444, 0, 0, 555), np.array([0, 1, 0, 0, 1], bool)),     # env 1 again before its episode ends
      9: (lv(-1, -1, -1, 777, -1), np.array([1, 0, 1, 1, 0], bool)),   # back to -1 (envs 0, 2), env 3 a level
      10: (lv(-1, -1, -1, 888, -1), np.array([0, 0, 0, 1, 0], bool)),  # and once more before it ends
  }
  for t in range(22):
    if t in schedule:
      run.set_levels(*schedule[t])
    run.step(t, KINDS[t % 3])
  seeds = run.reached['seeds']
  assert {111, 333, 444, 555, 888} <= seeds, seeds
  assert not {222, 777, 0} & seeds, seeds  # assignments replaced before their episode started, or masked out


def test_set_levels_before_the_first_reset():
  K, seed = 3, 5
  run = Run(K=K, seed=seed, length=3)
  run.set_levels(np.array([99, -1, 2 ** 31 - 2], np.int32))
  run.reset()
  for t in range(10):
    run.step(t, KINDS[t % 3])
  assert run.reached['episodes'] >= 6


def test_reset_with_levels_without_auto_reset():
  """reset(mask, levels) on a batch without auto-reset: the masked envs start their level now, the others go on."""
  K, seed = 4, 17
  env = SimtLevelsEnv(num_envs=K, seed=seed, length=6)
  ora = OracleLevels(K, seed, length=6)
  obs = env.reset()
  for i in range(K):
    assert (obs[i] == ora.reset(i)).all()
  rs = np.random.RandomState(1)
  for t in range(14):
    if t in (3, 8):
      mask = np.array([1, t == 8, 0, 1], bool)
      levels = np.array([1000 + t, 2000 + t, 3000, -1 if t == 8 else 5], np.int32)
      ora.set_levels(levels, mask)
      obs = env.reset(mask, levels).copy()
      for i in np.flatnonzero(mask):
        assert parity.frame_problem(obs[i], ora.reset(i)) is None, (t, i)
    actions = rs.randint(0, 17, K)
    obs, reward, done = env.step(actions)
    finished = []
    for i, ref in enumerate(ora.refs):
      o, r, d = ref.step(int(actions[i]))
      assert np.float32(r) == reward[i] and d == bool(done[i]), (t, i)
      assert parity.frame_problem(obs[i], o) is None, (t, i)
      assert canon.diff(ref.export_state(), env.snapshot(i)) is None, (t, i)
      assert env.world_seed()[i] == ora.ws[i], (t, i)
      if d:
        assert env.final_world_seed[i] == ora.ws[i], (t, i)
        finished.append(i)
    if finished:
      mask = np.zeros(K, bool)
      mask[finished] = True
      obs = env.reset(mask).copy()
      for i in finished:
        assert parity.frame_problem(obs[i], ora.reset(i)) is None, (t, i)
        assert env.world_seed()[i] == ora.ws[i], (t, i)
  assert (env.level == ora.level).all()


# ---- 4. replay a logged episode ---------------------------------------------------------------------------
def test_replay_a_logged_episode_from_its_final_world_seed():
  """Batch A (default levels, auto-reset) logs info['final_world_seed'] and the actions of an episode that is not
  its env's first; batch B (another seed) replays them on another env index as a level: the same obs, reward,
  done and canonical state at every step."""
  K, seed, length = 3, 23, 7
  a = SimtLevelsEnv(num_envs=K, seed=seed, length=length, auto_reset=True)
  a.reset()
  rs = np.random.RandomState(9)
  i = 1
  log, episode = [], 0
  cur = dict(first_obs=a.obs[i].copy(), first_state=a.snapshot(i), steps=[])
  while episode < 2:
    actions = rs.randint(0, 17, K).astype(np.int32)
    obs, reward, done = a.step(actions)
    d = bool(done[i])
    cur['steps'].append(dict(action=int(actions[i]), reward=reward[i], done=d,
                             obs=(a.final_obs[i] if d else obs[i]).copy(), state=None if d else a.snapshot(i)))
    if d:
      cur['seed'] = int(a.final_world_seed[i])
      log.append(cur)
      episode += 1
      cur = dict(first_obs=obs[i].copy(), first_state=a.snapshot(i), steps=[])
  ep = log[1]
  assert ep['seed'] == world_seed(seed + i, 2)
  b = SimtLevelsEnv(num_envs=2, seed=seed + 500, length=length)
  levels = np.array([-1, ep['seed']], np.int32)
  obs = b.reset(levels=levels)
  assert (obs[1] == ep['first_obs']).all() and canon.diff(ep['first_state'], b.snapshot(1)) is None
  for t, s in enumerate(ep['steps']):
    obs, reward, done = b.step(np.array([0, s['action']], np.int32))
    assert reward[1] == s['reward'] and bool(done[1]) == s['done'], t
    assert parity.frame_problem(obs[1], s['obs']) is None, t
    if s['state'] is not None:
      assert canon.diff(s['state'], b.snapshot(1)) is None, t
  assert s['done']


# ---- the oracle's levels ------------------------------------------------------------------------------
@pytest.mark.parametrize('episode', [1, 3])
def test_oracle_level_equals_the_oracle_on_that_world(episode):
  """tests/oracle_levels: an oracle env on level world_seed(s0, e) plays what the oracle env of seed s0 plays in
  its episode e -- state, frames, reward and done -- though its own seed and episode counter differ."""
  from oracle import oracle_env
  s0, length = 41, 30
  plain = oracle_env.OracleEnv(seed=s0, length=length)
  plain.set_episode(episode - 1)
  want = plain.reset()
  lev = oracle_levels.LevelEnv(seed=900, length=length)
  lev.set_level(world_seed(s0, episode))
  got = lev.reset()
  assert lev.world_seed == world_seed(s0, episode) and lev.episode == 1
  rs = np.random.RandomState(episode)
  for t in range(40):
    assert parity.frame_problem(got, want) is None, (t, parity.frame_problem(got, want))
    assert canon.diff(plain.export_state(), lev.export_state()) is None, t
    a = int(rs.randint(0, 17))
    want, r0, d0 = plain.step(a)
    got, r1, d1 = lev.step(a)
    assert (r0, d0) == (r1, d1), t
  lev.set_level(-1)
  lev.reset()
  assert lev.world_seed == world_seed(900, 2)


# ---- 5. errors and plumbing ----------------------------------------------------------------------------------
def test_levels_are_checked_on_the_host():
  B = 4
  ok = np.array([-1, 0, MAX_LEVEL, 5], np.int32)
  arr, mask = check_levels(ok, None, B)
  assert arr.tolist() == ok.tolist() and mask is None
  for bad in ([-2, 0, 0, 0], [0, 0, 0, MAX_LEVEL + 1], np.array([0, 0, 0, 2 ** 32 - 1], np.uint32)):
    with pytest.raises(ValueError, match='world seeds'):
      check_levels(np.asarray(bad) if not isinstance(bad, list) else np.array(bad, np.int64), None, B)
  with pytest.raises(ValueError, match='shape'):
    check_levels(np.zeros(B + 1, np.int32), None, B)
  with pytest.raises(ValueError, match='shape'):
    check_levels(np.zeros((B, 1), np.int32), None, B)
  with pytest.raises(ValueError, match='shape'):
    check_levels(ok, np.ones(B - 1, bool), B)
  import torch
  for dtype in (np.float32, np.float64, bool):
    with pytest.raises(ValueError, match='integers'):
      check_levels(np.zeros(B, dtype), None, B)
  with pytest.raises(ValueError, match='integers'):
    check_levels(torch.zeros(B), None, B)
  # entries outside the mask are ignored
  arr, mask = check_levels(np.array([-7, 3, 2 ** 40, 1], np.int64), np.array([0, 1, 0, 1], bool), B)
  assert mask.tolist() == [False, True, False, True]


def test_set_levels_without_the_level_buffer_fails():
  env = SimtLevelsEnv(num_envs=2, seed=3, level_buffers=False)
  with pytest.raises(RuntimeError, match='no level buffer'):
    env.set_levels(np.array([5, 5], np.int32))
  assert env.counters() == (0, 0)
  env.reset()  # the default sequence, untouched
  assert env.world_seed().tolist() == [world_seed(3, 1), world_seed(4, 1)]


def test_vector_env_passes_levels_through():
  calls = []

  class FakeEnv:
    _seed = 0

    def reset(self, mask=None, levels=None):
      calls.append(('reset', mask, levels))
      return np.zeros(1)

    def set_levels(self, levels, mask=None):
      calls.append(('set_levels', mask, levels))

  venv = vector.VectorEnv.__new__(vector.VectorEnv)
  venv.env, venv._to_numpy = FakeEnv(), False
  venv.reset(options={'levels': [3, 4]})
  venv.reset(options={'reset_mask': [1, 0], 'levels': [5, -1]})
  venv.set_levels([6, 7], mask=[0, 1])
  assert calls == [('reset', None, [3, 4]), ('reset', [1, 0], [5, -1]), ('set_levels', [0, 1], [6, 7])]


def test_abi_carries_the_level_buffers():
  names = [f[0] for f in _cabi.CrState._fields_]
  assert names[-2:] == ['level', 'final_world_seed'] and _cabi.ABI_VERSION == 6
  assert 'cr_set_levels' in _cabi.EXPORTS


def test_set_levels_kernel_does_not_spill(ptxas):  # noqa: F811
  found = {targs: v for (name, targs), v in ptxas.items() if name == 'k_set_levels'}
  assert len(found) == 1 and all(v.get('spill', 0) == 0 for v in found.values()), found
