"""observation='semantic' on the product's kernels on the SIMT emulator, against the C oracle: the step without
frames (cr_step_local: k_local in place of the frame kernel, k_final_local in place of k_terminal) and the
window of the state as it stands (cr_local).

The expected window is LocalView's crop (engine.py:165-176) of the oracle's info['semantic'] around the
player, restated below and padded with 0 outside the map.  The sweep runs every geometry of
tests/geometry_cases.py, and one whose map is smaller than the window on both axes, with the protocol of
tests/test_geometry_sweep.py: three envs from steps 150, 154 and 158 with a length of 160 (every env
truncates inside the run), inventory counts of 0, 1 to 9 and 10 or more, frequent 'sleep' actions, terminal
windows on.  Every step: windows, reward, done, canonical state, and the info entries 'facing', 'sleeping'
and 'daylight'; for ended envs the terminal window and terminal semantic map."""
import ctypes
import types

import numpy as np
import pytest
import torch

from crafter_b200 import recorder
from crafter_b200 import rules
from crafter_b200 import _cabi
from crafter_b200 import state as state_lib
from crafter_b200 import tables as tables_lib
from crafter_b200 import vector
from crafter_b200.env import FACING, daylight_at, player_facing
from oracle import canon
from tests import geometry_cases as gc
from tests import hostsim_env
from tests.test_build_properties import ptxas  # noqa: F401  (fixture)
from tests.test_geometry_sweep import LENGTH, boost
from tests.test_schedule_knobs import SLEEP, SLEEPING, _put

# the canonical player vector (oracle/canon.py): facing index, x, y
FACING_IDX, PX, PY = SLEEPING + 1, SLEEPING + 3, SLEEPING + 4
SIDES = ('left', 'right', 'top', 'bottom')
# the sweep's geometries and one whose map is smaller than the 9 x 7 window on both axes
CASES = {name: gc.kwargs(name) for name in gc.CASES}
CASES['map_smaller_than_window'] = dict(area=(7, 5), view=(9, 9), size=(64, 64))


def grid_of(view):
  """The local view (env.py:42-44): (view_w, view_h - item rows)."""
  return view[0], view[1] - -(-16 // view[0])


def expected_windows(semantic, px, py, grid):
  """LocalView's crop (engine.py:165-176) of info['semantic'] maps (N, W, H) around players at (px, py):
  (N, gx, gy) uint8, cell (x, y) = map cell player + (x, y) - grid // 2, 0 outside the map."""
  semantic = np.asarray(semantic)
  n, w, h = semantic.shape
  gx, gy = grid
  xs = np.asarray(px, np.int64)[:, None] + np.arange(gx) - gx // 2
  ys = np.asarray(py, np.int64)[:, None] + np.arange(gy) - gy // 2
  inside = ((xs >= 0) & (xs < w))[:, :, None] & ((ys >= 0) & (ys < h))[:, None, :]
  cells = semantic[np.arange(n)[:, None, None], xs.clip(0, w - 1)[:, :, None], ys.clip(0, h - 1)[:, None, :]]
  return np.where(inside, cells, 0).astype(np.uint8)


def clipped_sides(px, py, grid, area):
  """The sides of the map a window around (px, py) reaches past."""
  x0, y0 = px - grid[0] // 2, py - grid[1] // 2
  return {s for s, c in zip(SIDES, (x0 < 0, x0 + grid[0] > area[0], y0 < 0, y0 + grid[1] > area[1])) if c}


def window_problem(got, want):
  """First difference of two windows (gx, gy), or None."""
  bad = np.argwhere(got != want)
  if not len(bad):
    return None
  x, y = bad[0]
  return f'{len(bad)} cells differ, first at (x={x}, y={y}): {int(got[x, y])} vs oracle {int(want[x, y])}'


_LOCAL_LIB = []


def simt_local_lib():
  """tests/simt/simt_local.cpp: the SIMT emulator's kernels and step (simt_env.cpp) plus hs_step_local,
  hs_local and hs_set_final_local; the C interface of hostsim_env.simt_lib() otherwise."""
  if not _LOCAL_LIB:
    here = hostsim_env.HERE
    src = here / 'simt' / 'simt_local.cpp'
    out = here / 'simt' / '_build' / 'libsimt_local.so'
    deps = [src, here / 'simt' / 'simt_env.cpp', here / 'simt' / 'simt.h'] + list(
        (here.parent / 'crafter_b200' / 'csrc').glob('*.h')) + [here.parent / 'include' / 'crafter_b200.h']
    hostsim_env._compile(out, src, deps)
    L = ctypes.CDLL(str(out))
    vp = ctypes.c_void_p
    L.hs_create.argtypes = [ctypes.POINTER(_cabi.CrConfig), ctypes.POINTER(_cabi.CrTables),
                            ctypes.POINTER(_cabi.CrState), ctypes.POINTER(vp)]
    L.hs_destroy.argtypes = [vp]
    L.hs_reset.argtypes = [vp, vp, vp]
    L.hs_step.argtypes = [vp] * 5
    L.hs_render.argtypes = [vp, vp]
    L.hs_semantic.argtypes = [vp, vp]
    L.hs_last_error.restype = ctypes.c_char_p
    L.hs_step_local.argtypes = [vp] * 5
    L.hs_local.argtypes = [vp, vp]
    L.hs_set_final_local.argtypes = [vp] * 3
    _LOCAL_LIB.append(L)
  return _LOCAL_LIB[0]


class SimtRgbEnv(hostsim_env.SimtEnv):
  """SimtEnv on simt_local_lib(): frame steps (hs_step), and cr_local through local_semantic_of()."""

  def __init__(self, **kwargs):
    super().__init__(**kwargs)
    view = kwargs.get('view', (9, 9))
    self.grid = tuple(int(v) for v in tables_lib.geometry(view, kwargs.get('size', (64, 64)))['grid'])

  @staticmethod
  def _load(max_obj_tiles):
    assert max_obj_tiles is None
    return simt_local_lib()


class SimtLocalEnv(SimtRgbEnv):
  """observation='semantic' on the emulator: reset() is cr_reset without a frame followed by cr_local, step()
  is cr_step_local (hs_reset, hs_local, hs_step_local of tests/simt/simt_local.cpp); final_obs asks for
  terminal windows and terminal semantic maps (cr_state.final_local, final_semantic)."""

  def __init__(self, final_obs=False, **kwargs):
    super().__init__(**kwargs)
    self.local = np.zeros((self.B,) + self.grid, np.uint8)
    self.final_local = np.zeros((self.B,) + self.grid, np.uint8) if final_obs else None
    if final_obs:
      self.final_semantic = np.zeros((self.B,) + self.area, np.uint8)
      self._L.hs_set_final_local(self.h, self.final_local.ctypes.data, self.final_semantic.ctypes.data)

  def reset(self, mask=None):
    m = None if mask is None else np.ascontiguousarray(mask, np.uint8)
    self._L.hs_reset(self.h, None if m is None else m.ctypes.data, None)
    self._L.hs_local(self.h, self.local.ctypes.data)
    return self.local

  def step(self, actions):
    a = np.ascontiguousarray(actions, np.int32)
    self._L.hs_step_local(self.h, a.ctypes.data, self.local.ctypes.data, self.reward.ctypes.data,
                          self.done.ctypes.data)
    return self.local, self.reward, self.done.astype(bool)


def local_semantic_of(env):
  """cr_local (hs_local) of a SimtEnv of either kind: the window of every env as the state stands."""
  out = np.zeros((env.B,) + env.grid, np.uint8)
  env._L.hs_local.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
  env._L.hs_local(env.h, out.ctypes.data)
  return out


def oracle_window(ref, grid):
  st = ref.export_state()
  return st, expected_windows(ref.semantic()[None], [st['player'][PX]], [st['player'][PY]], grid)[0]


def check_info_entries(where, env, refs, states):
  """'facing', 'sleeping' and 'daylight' of crafter_b200.Env from the env's state tensors, against the oracle."""
  ents, pstate = torch.from_numpy(env.state['ents']), torch.from_numpy(env.state['pstate'])
  facing = player_facing(ents).numpy()
  daylight = daylight_at(pstate, torch.from_numpy(env.tables['daylight'])).numpy()
  sleeping = (pstate[:, 4] != 0).numpy()
  from oracle import oracle_env
  table = oracle_env.daylight_table(LENGTH + 2)
  for i, st in enumerate(states):
    player = st['player']
    assert tuple(facing[i]) == FACING[player[FACING_IDX]], where + (i, 'facing', facing[i], player[FACING_IDX])
    assert bool(sleeping[i]) == bool(player[SLEEPING]), where + (i, 'sleeping')
    step = int(env.state['pstate'][i, 9])
    assert daylight[i] == np.float32(table[step]) == np.float32(st['daylight']), where + (i, 'daylight', daylight[i])


def check_windows_against_oracle(make_env, K=3, steps=16, seed=70, length=LENGTH, **geometry):
  """The protocol of tests/test_geometry_sweep.run_case in semantic mode; returns what the run reached."""
  from oracle import oracle_env
  grid = grid_of(geometry.get('view', (9, 9)))
  area = geometry.get('area', (64, 64))
  env = make_env(num_envs=K, seed=seed, length=length, auto_reset=True, final_obs=True, **geometry)
  refs = [oracle_env.OracleEnv(seed=seed + i, length=length, **geometry) for i in range(K)]
  reached = dict(episodes=0, terminal_windows=0, windows=0, clipped=set())
  local = np.asarray(env.reset()).copy()
  for i, ref in enumerate(refs):
    ref.reset()
    problem = window_problem(local[i], oracle_window(ref, grid)[1])
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
    local, reward, done = env.step(actions)
    states = []
    for i, ref in enumerate(refs):
      where = (t, i)
      r, d = ref.step_norender(int(actions[i]))
      assert np.float32(r) == reward[i] and d == bool(done[i]), where + ('reward / done',)
      if d:
        st, want = oracle_window(ref, grid)
        problem = window_problem(env.final_local[i], want)
        assert problem is None, where + ('terminal window', problem)
        assert (env.final_semantic[i] == ref.semantic()).all(), where + ('terminal semantic',)
        reached['terminal_windows'] += 1
        reached['clipped'] |= clipped_sides(st['player'][PX], st['player'][PY], grid, area)
        ref.reset()
        reached['episodes'] += 1
      st, want = oracle_window(ref, grid)
      problem = canon.diff(st, env.snapshot(i))
      assert problem is None, where + (problem,)
      problem = window_problem(local[i], want)
      assert problem is None, where + ('window', problem)
      reached['windows'] += 1
      reached['clipped'] |= clipped_sides(st['player'][PX], st['player'][PY], grid, area)
      states.append(st)
    check_info_entries((t,), env, refs, states)
  semantic = env.semantic()
  for i, ref in enumerate(refs):
    assert (ref.semantic() == semantic[i]).all(), ('semantic', i)
  return reached


@pytest.mark.parametrize('name', list(CASES))
def test_semantic_geometry_sweep(name):
  """Terminal windows are compared at every geometry, the two where terminal frames are rejected
  (unstaged_256, no_tile_cache_512) included."""
  K = 3
  reached = check_windows_against_oracle(SimtLocalEnv, K=K, **CASES[name])
  assert reached['episodes'] >= K, (name, 'an env did not truncate', reached)
  assert reached['terminal_windows'] >= K, (name, 'too few terminal windows compared', reached)
  if name == 'map_smaller_than_window':
    assert reached['clipped'] == set(SIDES), (name, reached)
  print(name, {k: sorted(v) if isinstance(v, set) else v for k, v in reached.items()})


def test_sweep_has_terminal_windows_where_frames_are_rejected():
  rejected = {name for name in gc.CASES if not gc.geom(name)['terminal_ok']}
  assert {'unstaged_256', 'no_tile_cache_512'} <= rejected <= set(CASES), rejected


def test_windows_clipped_on_every_side_at_the_default_area():
  """Players walked to each edge of a 64 x 64 map (state written on both sides): the window of the default
  geometry clipped on each side, alone and at the corners."""
  from oracle import oracle_env
  grid, K = grid_of((9, 9)), 6
  env = SimtLocalEnv(num_envs=K, seed=5)
  env.reset()
  spots = [(0, 30), (63, 30), (30, 0), (30, 63), (1, 62), (62, 2)]
  seen = set()
  for i, (x, y) in enumerate(spots):
    ref = oracle_env.OracleEnv(seed=5 + i)
    ref.reset()
    st = ref.export_state()
    st['objs'] = st['objs'][st['objs'][:, 0] == 1]  # the player alone, moved to (x, y)
    st['objs'][0, 1:3] = (x, y)
    st['player'][PX], st['player'][PY] = x, y
    ref.import_state(st, 0, 1, oracle_env.world_seed(5 + i, 1))
    objmap = env.state['objmap'][i]
    ents = env.state['ents'][i].view(state_lib.ENT_DTYPE)
    live = np.flatnonzero(ents['type'][2:int(env.state['pstate'][i, 8])] != 0) + 2
    for slot in live:
      objmap[int(ents['x'][slot]) * 64 + int(ents['y'][slot])] = 0
      ents['type'][slot] = 0
    px, py = int(env.state['pstate'][i, 12]), int(env.state['pstate'][i, 13])
    objmap[px * 64 + py] = 0
    objmap[x * 64 + y] = 1
    ents['x'][1], ents['y'][1] = x, y
    env.state['pstate'][i, 12:14] = (x, y)
    env.state['mat'][i] = ref.export_state()['mat'].reshape(-1)
    got = local_semantic_of(env)[i]
    want = expected_windows(ref.semantic()[None], [x], [y], grid)[0]
    assert window_problem(got, want) is None, (x, y, window_problem(got, want))
    seen |= clipped_sides(x, y, grid, (64, 64))
  assert seen == set(SIDES), seen


def test_reset_mask_windows():
  """reset(mask) between auto-resets: the windows of the reset envs are the first of their new episode, the
  others those of the state as it stands."""
  from oracle import oracle_env
  K, seed, length = 4, 90, 3
  grid = grid_of((9, 9))
  env = SimtLocalEnv(num_envs=K, seed=seed, length=length, auto_reset=True)
  refs = [oracle_env.OracleEnv(seed=seed + i, length=length) for i in range(K)]
  local = np.asarray(env.reset()).copy()
  for i, ref in enumerate(refs):
    ref.reset()
    assert window_problem(local[i], oracle_window(ref, grid)[1]) is None, ('reset', i)
  rs = np.random.RandomState(5)
  for t in range(13):
    if t in (2, 3, 7):
      mask = np.array([t % 2 == 0, True, False, t == 7])
      local = np.asarray(env.reset(mask)).copy()
      for i in np.flatnonzero(mask):
        refs[i].reset()
      for i, ref in enumerate(refs):
        st, want = oracle_window(ref, grid)
        assert canon.diff(st, env.snapshot(i)) is None, (t, i)
        assert window_problem(local[i], want) is None, (t, i, 'reset(mask)', window_problem(local[i], want))
    actions = rs.randint(0, 17, K).astype(np.int32)
    local, reward, done = env.step(actions)
    for i, ref in enumerate(refs):
      r, d = ref.step_norender(int(actions[i]))
      assert d == bool(done[i]) and np.float32(r) == reward[i], (t, i)
      if d:
        ref.reset()
      st, want = oracle_window(ref, grid)
      assert canon.diff(st, env.snapshot(i)) is None, (t, i)
      assert window_problem(local[i], want) is None, (t, i, window_problem(local[i], want))


@pytest.mark.parametrize('name', ['default', 'view5x7', 'wide_area'])
def test_local_semantic_after_rgb_steps(name):
  """cr_local after frame steps (cr_step) on the same kind of handle: the window Env.local_semantic() and
  info['local_semantic'] return in 'rgb' mode, against the oracle and against the crop of info['semantic']."""
  from oracle import oracle_env
  geometry = gc.kwargs(name)
  grid = grid_of(geometry['view'])
  K, seed = 3, 21
  env = SimtRgbEnv(num_envs=K, seed=seed, auto_reset=True, **geometry)
  refs = [oracle_env.OracleEnv(seed=seed + i, **geometry) for i in range(K)]
  env.reset()
  for ref in refs:
    ref.reset()
  rs = np.random.RandomState(2)
  for t in range(6):
    actions = rs.randint(0, 17, K).astype(np.int32)
    obs = env.step(actions)[0].copy()
    got = local_semantic_of(env)
    assert (env.obs == obs).all(), 'cr_local changed the frames'
    pos = env.state['pstate'][:, 12:14]
    assert (got == expected_windows(env.semantic(), pos[:, 0], pos[:, 1], grid)).all(), t
    for i, ref in enumerate(refs):
      if ref.step_norender(int(actions[i]))[1]:
        ref.reset()
      problem = window_problem(got[i], oracle_window(ref, grid)[1])
      assert problem is None, (t, i, problem)


def test_episode_recorder_needs_frames(tmp_path):
  env = types.SimpleNamespace(observation='semantic', _auto_reset=False)
  with pytest.raises(ValueError, match="observation='semantic'"):
    recorder.EpisodeRecorder(env, tmp_path)
  with pytest.raises(ValueError, match='image'):
    recorder.Recorder(env, tmp_path, save_stats=False, save_video=False)


def test_vector_spaces_of_semantic_windows():
  single, single_act, batched, batched_act = vector._spaces(5, grid_of((9, 9)), 17, 18)
  assert tuple(single.shape) == (9, 7) and tuple(batched.shape) == (5, 9, 7)
  assert int(np.max(single.high)) == 18 and int(np.min(single.low)) == 0 and single.dtype == np.uint8
  assert single.contains(np.full((9, 7), 18, np.uint8)) and not single.contains(np.full((9, 7), 19, np.uint8))
  assert single_act.n == 17


def test_new_kernels_do_not_spill(ptxas):  # noqa: F811
  """k_local and k_final_local: 0 spill bytes in every instantiation (ptxas.log)."""
  for kernel in ('k_local', 'k_final_local'):
    found = {targs: v for (name, targs), v in ptxas.items() if name == kernel}
    assert len(found) == 2, (kernel, found)
    assert all(v.get('spill', 0) == 0 for v in found.values()), (kernel, found)
