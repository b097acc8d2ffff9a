"""ORACLE: ctypes front-end of oracle/crafter_oracle.c (single env, CPU).  Test infrastructure."""
import ctypes
import pathlib

import numpy as np
from PIL import Image

from oracle import build as _build

ATLAS = pathlib.Path(__file__).resolve().parents[1] / 'crafter_b200' / 'assets' / 'atlas16.npz'

MATERIALS = ['water', 'grass', 'stone', 'path', 'sand', 'tree', 'lava', 'coal', 'iron', 'diamond',
             'table', 'furnace']  # data.yaml:20-32
ITEMS = ['health', 'food', 'drink', 'energy', 'sapling', 'wood', 'stone', 'coal', 'iron', 'diamond',
         'wood_pickaxe', 'stone_pickaxe', 'iron_pickaxe', 'wood_sword', 'stone_sword',
         'iron_sword']  # data.yaml:39-55
ACHIEVEMENTS = [
    'collect_coal', 'collect_diamond', 'collect_drink', 'collect_iron', 'collect_sapling',
    'collect_stone', 'collect_wood', 'defeat_skeleton', 'defeat_zombie', 'eat_cow', 'eat_plant',
    'make_iron_pickaxe', 'make_iron_sword', 'make_stone_pickaxe', 'make_stone_sword',
    'make_wood_pickaxe', 'make_wood_sword', 'place_furnace', 'place_plant', 'place_stone',
    'place_table', 'wake_up']  # data.yaml:80-102
OBJ_TEXTURES = ['player-left', 'player-right', 'player-up', 'player-down', 'player-sleep', 'cow',
                'zombie', 'skeleton', 'arrow-left', 'arrow-right', 'arrow-up', 'arrow-down',
                'plant', 'plant-ripe']

_lib = None


def lib():
  global _lib
  if _lib is None:
    L = ctypes.CDLL(str(_build.ensure()))
    L.co_create.restype = ctypes.c_void_p
    L.co_create.argtypes = [ctypes.c_int] * 8 + [ctypes.c_int64]
    for name in ('co_destroy', 'co_reset'):
      getattr(L, name).argtypes = [ctypes.c_void_p]
    L.co_step.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    L.co_render.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    L.co_set_tables.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 6 + [ctypes.c_void_p] * 8 + [
        ctypes.c_int]
    L.co_set_episode.argtypes = [ctypes.c_void_p, ctypes.c_int64]
    L.co_set_inventory.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
    L.co_num_objects.argtypes = [ctypes.c_void_p]
    for name in ('co_export_objects', 'co_export_mat', 'co_export_player', 'co_export_touched',
                 'co_semantic'):
      getattr(L, name).argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    L.co_daylight.restype = ctypes.c_double
    L.co_daylight.argtypes = [ctypes.c_void_p]
    L.co_step_count.argtypes = [ctypes.c_void_p]
    L.co_rng_draws.restype = ctypes.c_long
    L.co_rng_draws.argtypes = [ctypes.c_void_p]
    L.co_world_seed.restype = ctypes.c_int64
    L.co_world_seed.argtypes = [ctypes.c_int64, ctypes.c_int64]
    L.co_run_random.argtypes = [
        ctypes.c_void_p, ctypes.c_int, ctypes.c_uint32, ctypes.c_int, ctypes.c_void_p]
    _lib = L
  return _lib


class Sprites:
  """Restates engine.py:120-142 (`Textures`): transposed originals + PIL NEAREST resizes."""

  def __init__(self):
    data = np.load(ATLAS)
    self._orig = {k: data[k].transpose((1, 0, 2)) for k in data.files}  # engine.py:126

  def get(self, name, size):
    size = int(size[0]), int(size[1])  # engine.py:134
    image = self._orig['unknown' if name is None else name]
    if image.shape[:2] == size:
      return image
    return np.array(Image.fromarray(image).resize(size[::-1], resample=Image.NEAREST))

  def rgba(self, name, size):
    tex = self.get(name, size)
    if tex.shape[-1] == 3:
      tex = np.concatenate([tex, np.full(tex.shape[:2] + (1,), 255, np.uint8)], -1)
    return np.ascontiguousarray(tex)


def daylight_table(n):
  """env.py:135-139 evaluated with the same numpy expressions, for step = 0..n-1."""
  out = np.zeros(n, np.float64)
  for step in range(n):
    progress = (step / 300) % 1 + 0.3
    out[step] = 1 - np.abs(np.cos(np.pi * progress)) ** 3
  return out


_DAY_CACHE = {}


def _daylight_cached(n):
  if n not in _DAY_CACHE:
    _DAY_CACHE[n] = daylight_table(n)
  return _DAY_CACHE[n]


def vignette(shape, stddev=0.5):
  """engine.py:213-218."""
  xs, ys = np.meshgrid(np.linspace(-1, 1, shape[0]), np.linspace(-1, 1, shape[1]))
  return np.ascontiguousarray(1 - np.exp(-0.5 * (xs ** 2 + ys ** 2) / (stddev ** 2)).T)


_TABLE_CACHE = {}


def render_tables(view, size):
  key = (tuple(int(v) for v in view), tuple(int(v) for v in size))
  if key not in _TABLE_CACHE:
    _TABLE_CACHE[key] = _render_tables(*key)
  return _TABLE_CACHE[key]


def _render_tables(view, size):
  view, size = np.array(view), np.array(size)
  unit = size // view  # env.py:122
  item_rows = int(np.ceil(len(ITEMS) / view[0]))  # env.py:42
  grid = np.array([view[0], view[1] - item_rows])
  igrid = np.array([view[0], item_rows])
  sp = Sprites()
  ux, uy = int(unit[0]), int(unit[1])
  mat = np.zeros((13, ux, uy, 3), np.uint8)
  for i, name in enumerate(MATERIALS):
    mat[i + 1] = sp.get(name, unit)[..., :3]  # engine.py:270-274 drops alpha
  obj = np.stack([sp.rgba(name, unit) for name in OBJ_TEXTURES])
  isz, dsz = 0.8 * unit, 0.6 * unit  # engine.py:240,247
  item = np.stack([sp.rgba(name, isz) for name in ITEMS])
  digit = np.stack([sp.rgba('unknown' if d == 0 else str(d), dsz) for d in range(10)])
  item_pos = np.zeros((16, 2), np.int32)
  digit_pos = np.zeros((16, 2), np.int32)
  for index in range(16):
    pos = index % igrid[0], index // igrid[0]
    item_pos[index] = (pos * unit + 0.1 * unit).astype(np.int32)  # engine.py:238-239
    digit_pos[index] = (pos * unit + 0.4 * unit).astype(np.int32)  # engine.py:244-245
  return dict(
      ux=ux, uy=uy, iw=item.shape[1], ih=item.shape[2], dw=digit.shape[1], dh=digit.shape[2],
      item_pos=item_pos, digit_pos=digit_pos, mat=mat, obj=obj, item=item, digit=digit,
      vignette=vignette(tuple(grid * unit)), grid=grid, item_rows=item_rows)


class OracleEnv:
  """Mirror of `crafter.Env` (env.py:25-118) on the C oracle."""

  def __init__(self, area=(64, 64), view=(9, 9), size=(64, 64), reward=True, length=10000, seed=0):
    view = tuple(view) if hasattr(view, '__len__') else (view, view)
    size = tuple(size) if hasattr(size, '__len__') else (size, size)
    self.area, self.view, self.size, self.length = tuple(area), view, size, length
    L = lib()
    self._h = L.co_create(area[0], area[1], view[0], view[1], size[0], size[1], int(length or 0),
                          int(bool(reward)), int(seed))
    t = render_tables(view, size)
    self._keep = t
    n_day = int(length or 0) + 2 if length else 100002
    day = _daylight_cached(n_day)
    L.co_set_tables(
        self._h, t['ux'], t['uy'], t['iw'], t['ih'], t['dw'], t['dh'],
        t['item_pos'].ctypes.data, t['digit_pos'].ctypes.data, t['mat'].ctypes.data,
        t['obj'].ctypes.data, t['item'].ctypes.data, t['digit'].ctypes.data,
        t['vignette'].ctypes.data, day.ctypes.data, n_day)
    self._obs = np.zeros((size[1], size[0], 3), np.uint8)

  def __del__(self):
    if getattr(self, '_h', None):
      lib().co_destroy(self._h)
      self._h = None

  def reset(self):
    lib().co_reset(self._h)
    return self.render()

  def step(self, action):
    r, d = ctypes.c_double(), ctypes.c_int()
    lib().co_step(self._h, int(action), ctypes.byref(r), ctypes.byref(d))
    return self.render(), r.value, bool(d.value)

  def step_norender(self, action):
    r, d = ctypes.c_double(), ctypes.c_int()
    lib().co_step(self._h, int(action), ctypes.byref(r), ctypes.byref(d))
    return r.value, bool(d.value)

  def render(self):
    lib().co_render(self._h, self._obs.ctypes.data)
    return self._obs.copy()

  def set_inventory(self, boost):
    for k, v in boost.items():
      lib().co_set_inventory(self._h, ITEMS.index(k), int(v))

  def set_episode(self, episode):
    lib().co_set_episode(self._h, int(episode))

  def semantic(self):
    out = np.zeros(self.area, np.uint8)
    lib().co_semantic(self._h, out.ctypes.data)
    return out

  def run_random(self, steps, policy_seed=0, render=True):
    return lib().co_run_random(self._h, int(steps), int(policy_seed), int(render),
                               self._obs.ctypes.data)

  def import_state(self, st, step, episode, world_seed):
    """Load a canonical state (oracle/canon.py) recorded from the reference (scenario fixtures)."""
    L = lib()
    c = lambda a, dt: np.ascontiguousarray(a, dt)
    mat, objs = c(st['mat'], np.uint8), c(st['objs'], np.int32)
    player, touched = c(st['player'], np.int64), c(st['touched'], np.int32)
    assert mat.shape == self.area and int(objs[0, 0]) == 1  # the player owns slot 1
    L.co_import_state.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                  ctypes.c_int, ctypes.c_int, ctypes.c_int64, ctypes.c_int64]
    L.co_import_state(self._h, mat.ctypes.data, objs.ctypes.data, len(objs), player.ctypes.data,
                      touched.ctypes.data, len(touched), int(step), int(episode), int(world_seed))

  def export_state(self):
    L = lib()
    n = L.co_num_objects(self._h)
    objs = np.zeros((n, 6), np.int32)
    L.co_export_objects(self._h, objs.ctypes.data)
    mat = np.zeros(self.area, np.uint8)
    L.co_export_mat(self._h, mat.ctypes.data)
    player = np.zeros(49, np.int64)
    L.co_export_player(self._h, player.ctypes.data)
    touched = np.zeros(4096, np.int32)
    nt = L.co_export_touched(self._h, touched.ctypes.data)
    return dict(mat=mat, objs=objs, player=player, touched=touched[:nt].copy(),
                daylight=L.co_daylight(self._h))


def world_seed(seed, episode):
  return lib().co_world_seed(int(seed), int(episode))


class OracleBatch:
  """N oracle envs stepped by a thread pool (CPU baseline of bench.py, full-batch parity test; env i
  has seed0 + i).  `threads` defaults to every host core.  Rendering is stateless (the night noise is
  keyed by the step), so skipping it with render=False changes nothing but the time taken."""

  def __init__(self, num_envs, threads=None, seed=0, **kwargs):
    import concurrent.futures
    import os
    self.envs = [OracleEnv(seed=seed + i, **kwargs) for i in range(num_envs)]
    self.n, self.threads = num_envs, max(1, min(threads or os.cpu_count() or 1, num_envs))
    self.size, self.area = self.envs[0].size, self.envs[0].area
    self.obs = np.zeros((num_envs, self.size[1], self.size[0], 3), np.uint8)
    self.reward = np.zeros(num_envs, np.float64)
    self.done = np.zeros(num_envs, np.int32)
    self._ptrs = (ctypes.c_void_p * num_envs)(*[e._h for e in self.envs])
    self._pool = concurrent.futures.ThreadPoolExecutor(self.threads)
    self._chunks = self._split(num_envs)
    L = lib()
    L.co_step_many.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                               ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    for name in ('co_reset_many', 'co_render_many', 'co_semantic_many', 'co_export_player_many'):
      getattr(L, name).argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]

  def _split(self, n):
    bounds = np.linspace(0, n, min(self.threads, max(n, 1)) + 1).astype(int)
    return [(int(a), int(b)) for a, b in zip(bounds[:-1], bounds[1:]) if b > a]

  def _ptr(self, a):
    return ctypes.addressof(self._ptrs) + a * ctypes.sizeof(ctypes.c_void_p)

  def _map(self, fn, ids, out):
    """fn(envs, n, out) over the envs `ids` (all when None) in parallel chunks; row k of `out`
    belongs to env ids[k]."""
    if ids is None:
      ptrs, n = self._ptrs, self.n
    else:
      ids = np.asarray(ids, np.int64).reshape(-1)
      ptrs, n = (ctypes.c_void_p * max(len(ids), 1))(*[self.envs[i]._h for i in ids]), len(ids)
    addr, step = ctypes.addressof(ptrs), ctypes.sizeof(ctypes.c_void_p)
    row = out[0].nbytes if out is not None and len(out) else 0
    data = out.ctypes.data if out is not None else None
    list(self._pool.map(lambda c: fn(addr + c[0] * step, c[1] - c[0],
                                     None if data is None else data + c[0] * row), self._split(n)))
    return out

  def reset(self, ids=None, render=True):
    """Start a new episode in every env (or in those of `ids`); with render, obs holds the frames."""
    out = None
    if render:
      out = self.obs if ids is None else np.zeros((len(ids),) + self.obs.shape[1:], np.uint8)
    self._map(lib().co_reset_many, ids, out)
    if render and ids is not None:
      self.obs[np.asarray(ids, np.int64)] = out
    return self.obs

  def step(self, actions, auto_reset=True, render=True):
    actions = np.ascontiguousarray(actions, np.int32)
    obs_stride = self.obs[0].nbytes
    list(self._pool.map(lambda c: lib().co_step_many(
        self._ptr(c[0]), c[1] - c[0], actions.ctypes.data + 4 * c[0],
        self.reward.ctypes.data + 8 * c[0], self.done.ctypes.data + 4 * c[0],
        self.obs.ctypes.data + c[0] * obs_stride if render else None, int(auto_reset)), self._chunks))
    return self.obs, self.reward, self.done.astype(bool)

  def render(self, ids=None):
    """Frames of the envs `ids` (all when None) as they stand: (len(ids), H, W, 3) uint8."""
    n = self.n if ids is None else len(ids)
    return self._map(lib().co_render_many, ids, np.zeros((n,) + self.obs.shape[1:], np.uint8))

  def semantic(self, ids=None):
    """info['semantic'] of the envs `ids` (all when None): (len(ids), W, H) uint8."""
    n = self.n if ids is None else len(ids)
    return self._map(lib().co_semantic_many, ids, np.zeros((n,) + tuple(self.area), np.uint8))

  def player(self, ids=None):
    """The 49-entry player vectors of oracle/canon.py of the envs `ids` (all when None): (len(ids), 49)."""
    n = self.n if ids is None else len(ids)
    return self._map(lib().co_export_player_many, ids, np.zeros((n, 49), np.int64))
