"""observation='symbolic' on the product's kernels on the SIMT emulator, against the C oracle: the step without
frames (cr_step_symbolic: k_symbolic in place of the frame kernel, k_final_local writing terminal vectors) and
the vector of the state as it stands (cr_symbolic).

The expected vector is a numpy restatement of its definition (include/crafter_b200.h, cr_step_symbolic) from
the oracle's canonical state (oracle/canon.py: mat, the objects with their type, position and `a` field, the
player vector) and the daylight table.  Every entry is 0, 1, k / 9 or a float32 rounding of a double, so
vectors are compared bit for bit.

The sweep runs every geometry of tests/test_semantic_obs.py with its protocol (three envs from steps 150, 154
and 158, length 160, boosted inventories, frequent 'sleep' actions, terminal outputs on).  Every step: vector,
reward, done, canonical state, and the window decoded from the vector against cr_local; for ended envs the
terminal vector and terminal semantic map.  The scenario fixtures (tests/golden/scenarios) replay in symbolic
mode against their recorded digests; their start states hold arrows of every facing and ripe plants."""
import ctypes
import functools
import pathlib
import types

import numpy as np
import pytest

from crafter_b200 import recorder
from crafter_b200 import rules
from crafter_b200 import state as state_lib
from crafter_b200 import vector
from crafter_b200.env import FACING, SYMBOLIC_CHANNELS, Env, symbolic_layout
from oracle import canon
from tests import hostsim_env
from tests import scenario_util as su
from tests.test_build_properties import ptxas  # noqa: F401  (fixture)
from tests.test_geometry_sweep import LENGTH, boost
from tests.test_schedule_knobs import SLEEP, SLEEPING, _put
from tests.test_semantic_obs import (CASES, FACING_IDX, PX, PY, SIDES, SimtLocalEnv, SimtRgbEnv, clipped_sides,
                                     grid_of, local_semantic_of)

SCEN = pathlib.Path(__file__).resolve().parent / 'golden' / 'scenarios'
GROUPS = sorted(p.stem for p in SCEN.glob('*.npz'))
N_MAT = len(rules.MATERIALS)
N_CH = len(SYMBOLIC_CHANNELS)
ARROW, PLANT = 5, 6  # canonical object types (oracle/canon.py)


# ---- the restatement ---------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _cell_xy(gx, gy):
  return np.meshgrid(np.arange(gx), np.arange(gy), indexing='ij')


def expected_vector(st, daylight, grid):
  """The symbolic vector of a canonical state `st` whose daylight is `daylight` (a float64), float32 (D,)."""
  mat, objs, player = np.asarray(st['mat']), np.asarray(st['objs']), np.asarray(st['player'])
  w, h = mat.shape
  gx, gy = grid
  x0, y0 = int(player[PX]) - gx // 2, int(player[PY]) - gy // 2
  cells = np.zeros((gx, gy, N_CH), np.float32)
  xs, ys = _cell_xy(gx, gy)
  wx, wy = xs + x0, ys + y0
  inside = (wx >= 0) & (wx < w) & (wy >= 0) & (wy < h)
  m = mat[wx.clip(0, w - 1), wy.clip(0, h - 1)].astype(np.int64)
  ok = inside & (m >= 1) & (m <= N_MAT)
  cells[xs[ok], ys[ok], m[ok] - 1] = 1
  kind, ox, oy, a = objs[:, 0], objs[:, 1] - x0, objs[:, 2] - y0, objs[:, 4]
  sel = (ox >= 0) & (ox < gx) & (oy >= 0) & (oy < gy)
  kind, a = kind[sel], a[sel]
  # the object channel (0..9 after the materials): arrows by facing, plants by ripeness (grown > 300,
  # objects.py:402-403), the others by type
  channel = np.where(kind == ARROW, 4 + a, np.where(kind == PLANT, np.where(a > 300, 9, 8), kind - 1))
  cells[ox[sel], oy[sel], N_MAT + channel] = 1
  inventory = np.asarray(player[:len(rules.ITEMS)], np.float32) / np.float32(9)
  facing = np.zeros(len(FACING), np.float32)
  facing[int(player[FACING_IDX])] = 1
  tail = np.array([player[SLEEPING] != 0, np.float32(daylight)], np.float32)
  return np.concatenate([cells.reshape(-1), inventory, facing, tail])


def vector_problem(got, want, grid):
  """First difference of two vectors, bit for bit, named by part (and cell and channel), or None."""
  got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
  if got.shape != want.shape:
    return f'shape {got.shape} vs {want.shape}'
  bad = np.flatnonzero(got.view(np.uint32) != want.view(np.uint32))
  if not len(bad):
    return None
  i = int(bad[0])
  part = next(p for p, s in symbolic_layout(grid).items() if s.start <= i < s.stop)
  at = f'{part}[{i - symbolic_layout(grid)[part].start}]'
  if part == 'map':
    c, ch = divmod(i, N_CH)
    at = f'map cell (x={c // grid[1]}, y={c % grid[1]}) channel {SYMBOLIC_CHANNELS[ch]}'
  return f'{len(bad)} entries differ, first {at}: {got[i]!r} vs expected {want[i]!r}'


def decode_window(vectors, grid):
  """The local semantic window (N, gx, gy) a batch of vectors shows: the object's id (13..18) where an object
  channel is set, else the material id, 0 where no channel is."""
  n = len(vectors)
  cells = np.asarray(vectors)[:, symbolic_layout(grid)['map']].reshape(n, grid[0], grid[1], N_CH) != 0
  mat = np.where(cells[..., :N_MAT].any(-1), cells[..., :N_MAT].argmax(-1) + 1, 0)
  obj_ids = 13 + np.array([0, 1, 2, 3, 4, 4, 4, 4, 5, 5])  # semantic ids: player .. arrow, plant (engine.py:253-258)
  obj = cells[..., N_MAT:]
  return np.where(obj.any(-1), obj_ids[obj.argmax(-1)], mat).astype(np.uint8)


class Coverage:
  """What the compared vectors showed: the cell channels set, facings, sleeping values, and whether an inventory
  entry was 9 (entry 1.0) and 0, each with the first case that showed it."""

  def __init__(self):
    self.seen = {}

  def add(self, case, vec, grid):
    lay = symbolic_layout(grid)
    cells = vec[lay['map']].reshape(-1, N_CH)
    keys = [f'channel {SYMBOLIC_CHANNELS[c]}' for c in np.flatnonzero(cells.any(0))]
    keys.append(f'facing {"left right up down".split()[int(np.argmax(vec[lay["facing"]]))]}')
    keys.append(f'sleeping {int(vec[lay["sleeping"]][0])}')
    inv = vec[lay['inventory']]
    keys += ['inventory 9'] * bool((inv == 1).any()) + ['inventory 0'] * bool((inv == 0).any())
    for k in keys:
      self.seen.setdefault(k, case)

  @staticmethod
  def wanted():
    return ([f'channel {c}' for c in SYMBOLIC_CHANNELS] + [f'facing {f}' for f in 'left right up down'.split()] +
            ['sleeping 0', 'sleeping 1', 'inventory 9', 'inventory 0'])


# ---- the emulator build ----------------------------------------------------------------------------
_SYM_LIB = []


def simt_symbolic_lib():
  """tests/simt/simt_symbolic.cpp: simt_local_lib() plus hs_step_symbolic, hs_symbolic and
  hs_set_final_symbolic."""
  if not _SYM_LIB:
    here = hostsim_env.HERE
    src = here / 'simt' / 'simt_symbolic.cpp'
    out = here / 'simt' / '_build' / 'libsimt_symbolic.so'
    deps = [src, here / 'simt' / 'simt_local.cpp', here / 'simt' / 'simt_env.cpp', here / 'simt' / 'simt.h'] + list(
        (here.parent / 'crafter_b200' / 'csrc').glob('*.h')) + [here.parent / 'include' / 'crafter_b200.h']
    hostsim_env._compile(out, src, deps)
    L = ctypes.CDLL(str(out))
    vp = ctypes.c_void_p
    L.hs_create.argtypes = [ctypes.POINTER(hostsim_env._cabi.CrConfig), ctypes.POINTER(hostsim_env._cabi.CrTables),
                            ctypes.POINTER(hostsim_env._cabi.CrState), ctypes.POINTER(vp)]
    L.hs_destroy.argtypes = [vp]
    L.hs_reset.argtypes = [vp, vp, vp]
    L.hs_step.argtypes = [vp] * 5
    L.hs_render.argtypes = [vp, vp]
    L.hs_semantic.argtypes = [vp, vp]
    L.hs_recount.argtypes = [vp]
    L.hs_last_error.restype = ctypes.c_char_p
    L.hs_step_local.argtypes = [vp] * 5
    L.hs_local.argtypes = [vp, vp]
    L.hs_set_final_local.argtypes = [vp] * 3
    L.hs_step_symbolic.argtypes = [vp] * 5
    L.hs_symbolic.argtypes = [vp, vp]
    L.hs_set_final_symbolic.argtypes = [vp] * 3
    _SYM_LIB.append(L)
  return _SYM_LIB[0]


def symbolic_of(env):
  """cr_symbolic (hs_symbolic) of an env on simt_symbolic_lib(): the vector of every env as the state stands."""
  out = np.zeros((env.B, symbolic_layout(env.grid)['daylight'].stop), np.float32)
  env._L.hs_symbolic(env.h, out.ctypes.data)
  return out


class _OnSymbolicLib:
  @staticmethod
  def _load(max_obj_tiles):
    assert max_obj_tiles is None
    return simt_symbolic_lib()


class SimtRgbSymEnv(_OnSymbolicLib, SimtRgbEnv):
  """Frame steps (hs_step) on the symbolic build."""


class SimtLocalSymEnv(_OnSymbolicLib, SimtLocalEnv):
  """Window steps (hs_step_local) on the symbolic build."""


class SimtSymbolicEnv(_OnSymbolicLib, SimtRgbEnv):
  """observation='symbolic' on the emulator: reset() is cr_reset without a frame followed by cr_symbolic, step()
  is cr_step_symbolic; final_obs asks for terminal vectors and terminal semantic maps (cr_state.final_symbolic,
  final_semantic)."""

  def __init__(self, final_obs=False, **kwargs):
    super().__init__(**kwargs)
    dim = symbolic_layout(self.grid)['daylight'].stop
    self.vec = np.zeros((self.B, dim), np.float32)
    self.final_symbolic = np.zeros((self.B, dim), np.float32) if final_obs else None
    if final_obs:
      self.final_semantic = np.zeros((self.B,) + self.area, np.uint8)
      self._L.hs_set_final_symbolic(self.h, self.final_symbolic.ctypes.data, self.final_semantic.ctypes.data)

  def reset(self, mask=None):
    m = None if mask is None else np.ascontiguousarray(mask, np.uint8)
    self._L.hs_reset(self.h, None if m is None else m.ctypes.data, None)
    self._L.hs_symbolic(self.h, self.vec.ctypes.data)
    return self.vec

  def step(self, actions):
    a = np.ascontiguousarray(actions, np.int32)
    self._L.hs_step_symbolic(self.h, a.ctypes.data, self.vec.ctypes.data, self.reward.ctypes.data,
                             self.done.ctypes.data)
    return self.vec, self.reward, self.done.astype(bool)


def oracle_vector(ref, grid):
  st = ref.export_state()
  return st, expected_vector(st, st['daylight'], grid)


# ---- the geometry sweep ---------------------------------------------------------------------------------
def check_vectors_against_oracle(K=3, steps=16, seed=70, length=LENGTH, coverage=None, case='', **geometry):
  """The protocol of tests/test_semantic_obs.check_windows_against_oracle in symbolic mode."""
  from oracle import oracle_env
  grid = grid_of(geometry.get('view', (9, 9)))
  area = geometry.get('area', (64, 64))
  env = SimtSymbolicEnv(num_envs=K, seed=seed, length=length, auto_reset=True, final_obs=True, **geometry)
  refs = [oracle_env.OracleEnv(seed=seed + i, length=length, **geometry) for i in range(K)]
  reached = dict(episodes=0, terminal_vectors=0, vectors=0, clipped=set())
  coverage = coverage if coverage is not None else Coverage()
  vec = env.reset().copy()
  for i, ref in enumerate(refs):
    ref.reset()
    problem = vector_problem(vec[i], oracle_vector(ref, grid)[1], grid)
    assert problem is None, ('reset', i, problem)
  counts = boost(K)
  for item, col in counts.items():
    _put(env.state['inventory'], rules.ITEMS.index(item), col)
    for i, ref in enumerate(refs):
      ref.set_inventory({item: int(col[i])})
  start = np.array([150 + 4 * i for i in range(K)], np.int32)
  _put(env.state['pstate'], state_lib.PS['step'], start)
  for i, ref in enumerate(refs):
    ref.import_state(ref.export_state(), int(start[i]), 1, oracle_env.world_seed(seed + i, 1))
  rs = np.random.RandomState(3)
  for t in range(steps):
    actions = rs.randint(0, 17, K).astype(np.int32)
    actions[rs.rand(K) < 0.35] = SLEEP
    vec, reward, done = env.step(actions)
    for i, ref in enumerate(refs):
      where = (case, t, i)
      r, d = ref.step_norender(int(actions[i]))
      assert np.float32(r) == reward[i] and d == bool(done[i]), where + ('reward / done',)
      if d:
        st, want = oracle_vector(ref, grid)
        problem = vector_problem(env.final_symbolic[i], want, grid)
        assert problem is None, where + ('terminal vector', problem)
        assert (env.final_semantic[i] == ref.semantic()).all(), where + ('terminal semantic',)
        coverage.add(case, want, grid)
        reached['terminal_vectors'] += 1
        reached['clipped'] |= clipped_sides(st['player'][PX], st['player'][PY], grid, area)
        ref.reset()
        reached['episodes'] += 1
      st, want = oracle_vector(ref, grid)
      problem = canon.diff(st, env.snapshot(i))
      assert problem is None, where + (problem,)
      problem = vector_problem(vec[i], want, grid)
      assert problem is None, where + ('vector', problem)
      coverage.add(case, want, grid)
      reached['vectors'] += 1
      reached['clipped'] |= clipped_sides(st['player'][PX], st['player'][PY], grid, area)
    local = local_semantic_of(env)
    assert (decode_window(vec, grid) == local).all(), (case, t, 'the decoded vector is not the window of cr_local')
  return reached


@pytest.mark.parametrize('name', list(CASES))
def test_symbolic_geometry_sweep(name):
  """Terminal vectors are compared at every geometry, the two where terminal frames are rejected included."""
  K = 3
  reached = check_vectors_against_oracle(K=K, case=name, **CASES[name])
  assert reached['episodes'] >= K, (name, 'an env did not truncate', reached)
  assert reached['terminal_vectors'] >= K, (name, 'too few terminal vectors compared', reached)
  if name == 'map_smaller_than_window':
    assert reached['clipped'] == set(SIDES), (name, reached)
  print(name, {k: sorted(v) if isinstance(v, set) else v for k, v in reached.items()})


# ---- the scenario fixtures -----------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def replay_symbolic(group):
  """The fixtures of `group` as one batch in symbolic mode: every step's state against the recorded digests and
  player vectors, reward and done against the recording, the vector against the restatement of the verified
  state (and the vector of the loaded start states through cr_symbolic).  Returns the Coverage."""
  from oracle import oracle_env
  z = np.load(SCEN / f'{group}.npz')
  K = int(z['meta_K'])
  names = [str(n) for n in z['meta_names']]
  kwargs = dict(area=tuple(int(v) for v in z['meta_area']), view=tuple(int(v) for v in z['meta_view']),
                size=tuple(int(v) for v in z['meta_size']), length=int(z['meta_length']))
  grid = grid_of(kwargs['view'])
  day = oracle_env.daylight_table(kwargs['length'] + 1026)
  env = SimtSymbolicEnv(num_envs=K, seed=int(z['meta_seed0']), auto_reset=False, **kwargs)
  env.reset()
  g = lambda i, k: z[f's{i}_{k}']
  steps = np.zeros(K, np.int64)
  for i in range(K):
    st = {k: g(i, k) for k in canon.KEYS}
    step, episode, world_seed = (int(v) for v in g(i, 'extras'))
    steps[i] = step
    su.load_numpy(env.state, i, su.raw_arrays(st, dict(step=step, episode=episode, world_seed=world_seed),
                                              kwargs['area'], env.state['ents'].shape[1]))
  env.recount()
  coverage = Coverage()
  vec = symbolic_of(env)
  for i in range(K):
    st = {k: g(i, k) for k in canon.KEYS}
    assert canon.diff(st, env.snapshot(i)) is None, (group, names[i], 'load')
    want = expected_vector(st, day[steps[i]], grid)
    assert vector_problem(vec[i], want, grid) is None, (group, names[i], 'load', vector_problem(vec[i], want, grid))
    coverage.add(f'{group}/{names[i]}', want, grid)
  n = [len(g(i, 'actions')) for i in range(K)]
  compared = 0
  for t in range(max(n)):
    actions = np.array([g(i, 'actions')[t] if t < n[i] else 0 for i in range(K)], np.int32)
    vec, reward, done = env.step(actions)
    steps += 1
    for i in range(K):
      if t >= n[i]:
        continue  # this scenario has ended (the reference env was done); its env idles on
      where = (group, names[i], t, int(actions[i]))
      snap = env.snapshot(i)
      assert (snap['player'] == g(i, 'player_t')[t]).all(), (where, 'player')
      for k, v in canon.digest(snap).items():
        assert v == int(g(i, f'{k}_crc')[t]), (where, k)
      assert reward[i] == np.float32(g(i, 'reward')[t]), (where, 'reward')
      assert bool(done[i]) == bool(g(i, 'done')[t]), (where, 'done')
      want = expected_vector(snap, day[steps[i]], grid)  # the state is the reference's: its digests matched
      problem = vector_problem(vec[i], want, grid)
      assert problem is None, (where, 'vector', problem)
      coverage.add(f'{group}/{names[i]}', want, grid)
      compared += 1
  assert compared == sum(n) and compared > 0
  return coverage


@pytest.mark.parametrize('group', GROUPS)
def test_symbolic_replays_scenarios(group):
  replay_symbolic(group)


def test_scenario_start_states_hold_every_arrow_facing_and_ripe_plants():
  facings, ripe = set(), 0
  for group in GROUPS:
    z = np.load(SCEN / f'{group}.npz')
    for i in range(int(z['meta_K'])):
      objs = z[f's{i}_objs']
      facings |= set(objs[objs[:, 0] == ARROW, 4].tolist())
      ripe += int(((objs[:, 0] == PLANT) & (objs[:, 4] > 300)).sum())
  assert facings == {0, 1, 2, 3} and ripe >= 11, (facings, ripe)


def test_symbolic_inputs_cover_every_channel():
  """Prints the channel -> case table over the vectors the scenario replays and the default sweep compare; fails
  when a cell channel, a facing, a sleeping value, or an inventory entry of 9 or 0 is never shown."""
  coverage = Coverage()
  for group in GROUPS:
    for k, case in replay_symbolic(group).seen.items():
      coverage.seen.setdefault(k, case)
  check_vectors_against_oracle(coverage=coverage, case='sweep default', **CASES['default'])
  for k in Coverage.wanted():
    print(f'  {k:24s} {coverage.seen.get(k, "MISSING")}')
  missing = [k for k in Coverage.wanted() if k not in coverage.seen]
  assert not missing, f'never shown by the compared vectors: {missing}'


def test_symbolic_values_at_their_edges():
  """States written directly, each next to its edge: plants grown 299, 300, 301 and 32767 and arrows of all four
  facings in view; inventory counts 0 to 47 (17, 25 and 34 are the counts where k * (1 / 9) and k / 9 round
  apart); every facing; sleeping; a step counter past the daylight table (clamped to its last entry)."""
  from oracle import oracle_env
  K, grid = 3, grid_of((9, 9))
  env = SimtSymbolicEnv(num_envs=K, seed=8, length=50)
  env.reset()
  n_day = len(env.tables['daylight'])
  ents = env.state['ents'].view(state_lib.ENT_DTYPE)
  ps, objmap, PS = env.state['pstate'], env.state['objmap'], state_lib.PS
  placed = [(6, 299), (6, 300), (6, 301), (6, 32767), (5, 0), (5, 1), (5, 2), (5, 3)]  # (type, aux)
  for i in range(K):
    px, py = int(ps[i, PS['player_x']]), int(ps[i, PS['player_y']])
    cells = [(px + dx, py + dy) for dy in (-2, 2) for dx in (-3, -1, 1, 3)]
    for (kind, aux), (x, y) in zip(placed, cells):
      old = int(objmap[i, x * 64 + y])
      if old:
        ents[i, old]['type'] = 0  # the occupant goes, as a tombstone
      slot = int(ps[i, PS['n_slots']])
      ents[i, slot] = (kind, 1, x, y, aux)
      objmap[i, x * 64 + y] = slot
      ps[i, PS['n_slots']] = slot + 1
    env.state['inventory'][i] = np.arange(16) + 16 * i
    ents[i, 1]['aux'] = i + 1
    ps[i, PS['sleeping']] = i % 2
  ps[2, PS['step']] = n_day + 5
  vec = symbolic_of(env)
  day = oracle_env.daylight_table(n_day)
  for i in range(K):
    want = expected_vector(env.snapshot(i), day[min(int(ps[i, PS['step']]), n_day - 1)], grid)
    assert vector_problem(vec[i], want, grid) is None, (i, vector_problem(vec[i], want, grid))
  lay = symbolic_layout(grid)
  cells = vec[:, lay['map']].reshape(K, -1, N_CH)
  for name in ('plant', 'plant-ripe', 'arrow-left', 'arrow-right', 'arrow-up', 'arrow-down'):
    assert (cells[:, :, SYMBOLIC_CHANNELS.index(name)].sum(1) >= 1).all(), name
  assert (cells[:, :, SYMBOLIC_CHANNELS.index('plant-ripe')].sum(1) >= 2).all()  # 301 and 32767, not 300
  assert vec[2, lay['daylight']][0] == np.float32(day[-1])


# ---- the other entry points --------------------------------------------------------------------------------
def test_layout():
  assert len(SYMBOLIC_CHANNELS) == 22 and SYMBOLIC_CHANNELS[:12] == tuple(rules.MATERIALS)
  lay = symbolic_layout(grid_of((9, 9)))
  assert lay['daylight'].stop == 1408 and lay['map'] == slice(0, 1386) and lay['inventory'] == slice(1386, 1402)
  assert lay['facing'] == slice(1402, 1406) and lay['sleeping'] == slice(1406, 1407)
  assert symbolic_layout(grid_of((15, 15)))['daylight'].stop == 22 * 15 * 13 + 22 == 4312


def test_reset_mask_vectors():
  """reset(mask) between auto-resets: the vectors of the reset envs are the first of their new episode, the
  others those of the state as it stands."""
  from oracle import oracle_env
  K, seed, length = 4, 90, 3
  grid = grid_of((9, 9))
  env = SimtSymbolicEnv(num_envs=K, seed=seed, length=length, auto_reset=True)
  refs = [oracle_env.OracleEnv(seed=seed + i, length=length) for i in range(K)]
  vec = env.reset().copy()
  for i, ref in enumerate(refs):
    ref.reset()
    assert vector_problem(vec[i], oracle_vector(ref, grid)[1], grid) is None, ('reset', i)
  rs = np.random.RandomState(5)
  for t in range(13):
    if t in (2, 3, 7):
      mask = np.array([t % 2 == 0, True, False, t == 7])
      vec = env.reset(mask).copy()
      for i in np.flatnonzero(mask):
        refs[i].reset()
      for i, ref in enumerate(refs):
        st, want = oracle_vector(ref, grid)
        assert canon.diff(st, env.snapshot(i)) is None, (t, i)
        assert vector_problem(vec[i], want, grid) is None, (t, i, 'reset(mask)', vector_problem(vec[i], want, grid))
    actions = rs.randint(0, 17, K).astype(np.int32)
    vec, reward, done = env.step(actions)
    for i, ref in enumerate(refs):
      r, d = ref.step_norender(int(actions[i]))
      assert d == bool(done[i]) and np.float32(r) == reward[i], (t, i)
      if d:
        ref.reset()
      st, want = oracle_vector(ref, grid)
      assert canon.diff(st, env.snapshot(i)) is None, (t, i)
      assert vector_problem(vec[i], want, grid) is None, (t, i, vector_problem(vec[i], want, grid))


@pytest.mark.parametrize('kind', ['rgb', 'semantic'])
@pytest.mark.parametrize('name', ['default', 'view5x7', 'wide_area'])
def test_symbolic_after_other_steps(kind, name):
  """cr_symbolic after frame steps (cr_step) and after window steps (cr_step_local) on the symbolic build, with
  terminal frames / windows on: Env.symbolic() in the other modes.  The frames and windows are left alone."""
  from oracle import oracle_env
  from tests import geometry_cases as gc
  geometry = gc.kwargs(name)
  grid = grid_of(geometry['view'])
  K, seed = 3, 21
  make = SimtRgbSymEnv if kind == 'rgb' else functools.partial(SimtLocalSymEnv, final_obs=True)
  env = make(num_envs=K, seed=seed, auto_reset=True, length=4, **geometry)
  refs = [oracle_env.OracleEnv(seed=seed + i, length=4, **geometry) for i in range(K)]
  env.reset()
  for ref in refs:
    ref.reset()
  rs = np.random.RandomState(2)
  for t in range(6):
    actions = rs.randint(0, 17, K).astype(np.int32)
    obs = env.step(actions)[0].copy()
    got = symbolic_of(env)
    assert (obs == (env.obs if kind == 'rgb' else env.local)).all(), 'cr_symbolic changed the obs'
    for i, ref in enumerate(refs):
      if ref.step_norender(int(actions[i]))[1]:
        ref.reset()
      problem = vector_problem(got[i], oracle_vector(ref, grid)[1], grid)
      assert problem is None, (t, i, problem)
    assert (decode_window(got, grid) == local_semantic_of(env)).all(), t


def test_recorder_and_step_host_need_frames(tmp_path):
  env = types.SimpleNamespace(observation='symbolic', _auto_reset=False)
  with pytest.raises(ValueError, match="observation='symbolic'"):
    recorder.EpisodeRecorder(env, tmp_path)
  with pytest.raises(ValueError, match='image'):
    recorder.Recorder(env, tmp_path, save_stats=False, save_video=False)
  with pytest.raises(RuntimeError, match="not available with observation='symbolic'"):
    Env.step_host(types.SimpleNamespace(_observation='symbolic'), None, None, None)


def test_vector_spaces_of_symbolic_vectors():
  single, single_act, batched, _ = vector._spaces(5, (1408,), 17, 1, np.float32)
  assert tuple(single.shape) == (1408,) and tuple(batched.shape) == (5, 1408) and single.dtype == np.float32
  assert single.contains(np.ones(1408, np.float32)) and not single.contains(np.full(1408, 2, np.float32))
  assert single.contains(single.sample()) and single_act.n == 17


def test_symbolic_kernels_do_not_spill(ptxas):  # noqa: F811
  """k_symbolic and the changed k_final_local: 0 spill bytes in every instantiation (ptxas.log)."""
  for kernel in ('k_symbolic', 'k_final_local'):
    found = {targs: v for (name, targs), v in ptxas.items() if name == kernel}
    assert len(found) == 2, (kernel, found)
    assert all(v.get('spill', 0) == 0 for v in found.values()), (kernel, found)
