"""TEST INFRASTRUCTURE: drives tests/hostsim (the device logic headers compiled for the host) with
numpy arrays, mirroring crafter_b200.Env closely enough to replay golden trajectories on a CPU-only
container.  Not a product path; crafter_b200 never imports this."""
import ctypes
import os
import pathlib
import subprocess

import numpy as np

from crafter_b200 import _cabi
from crafter_b200 import rules
from crafter_b200 import state as state_lib
from crafter_b200 import tables as tables_lib

HERE = pathlib.Path(__file__).resolve().parent
SRC = HERE / 'hostsim' / 'hostsim.cpp'
OUT = HERE / 'hostsim' / '_build' / 'libhostsim.so'

_libs = {}


def _compile(out, src, deps, extra=()):
  """g++ -> `out` when it is missing or older than `deps`; one builder at a time (pytest-xdist workers
  share the tree), and the library appears by rename so that nobody loads a half-written file."""
  import fcntl
  import os
  out.parent.mkdir(exist_ok=True)
  with open(out.parent / (out.name + '.lock'), 'w') as lock:
    fcntl.flock(lock, fcntl.LOCK_EX)
    if not out.exists() or any(d.stat().st_mtime > out.stat().st_mtime for d in deps):
      tmp = out.with_suffix(f'.tmp{os.getpid()}')
      subprocess.run(
          ['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-fno-fast-math', '-fPIC', '-shared',
           '-o', str(tmp), str(src), '-lm'] + list(extra), check=True)
      os.replace(tmp, out)


def lib(max_obj_tiles=None):
  """max_obj_tiles: build variant with a tiny object-tile cache (exercises the uncached path)."""
  global OUT
  key = max_obj_tiles
  if key not in _libs:
    OUT = HERE / 'hostsim' / '_build' / ('libhostsim.so' if key is None else f'libhostsim_t{key}.so')
    extra = [] if key is None else [f'-DCR_MAX_OBJ_TILES={key}']
    deps = [SRC] + list((HERE.parent / 'crafter_b200' / 'csrc').glob('*.h')) + [
        HERE.parent / 'include' / 'crafter_b200.h']
    _compile(OUT, SRC, deps, extra)
    L = ctypes.CDLL(str(OUT))
    vp = ctypes.c_void_p
    L.hs_create.argtypes = [ctypes.POINTER(_cabi.CrConfig), ctypes.POINTER(_cabi.CrTables),
                            ctypes.POINTER(_cabi.CrState), ctypes.POINTER(vp)]
    L.hs_destroy.argtypes = [vp]
    L.hs_reset.argtypes = [vp, vp, vp]
    L.hs_step.argtypes = [vp, vp, vp, vp, vp]
    L.hs_render.argtypes = [vp, vp]
    L.hs_semantic.argtypes = [vp, vp]
    L.hs_noise3.restype = ctypes.c_double
    L.hs_noise3.argtypes = [vp, ctypes.c_double, ctypes.c_double, ctypes.c_double]
    L.hs_last_error.restype = ctypes.c_char_p
    _libs[key] = L
  return _libs[key]


def simt_lib(max_obj_tiles=None):
  """tests/simt: the product's kernels (csrc/cr_kernels.h) on a SIMT emulator, same C interface.
  max_obj_tiles: build variant with a tiny object-tile cache, as lib()."""
  key = ('simt', max_obj_tiles)
  if key not in _libs:
    src = HERE / 'simt' / 'simt_env.cpp'
    out = HERE / 'simt' / '_build' / ('libsimt.so' if max_obj_tiles is None else f'libsimt_t{max_obj_tiles}.so')
    deps = [src, HERE / 'simt' / 'simt.h'] + list((HERE.parent / 'crafter_b200' / 'csrc').glob('*.h')) + [
        HERE.parent / 'include' / 'crafter_b200.h']
    _compile(out, src, deps, [] if max_obj_tiles is None else [f'-DCR_MAX_OBJ_TILES={max_obj_tiles}'])
    L = ctypes.CDLL(str(out))
    vp = ctypes.c_void_p
    L.hs_create.argtypes = [ctypes.POINTER(_cabi.CrConfig), ctypes.POINTER(_cabi.CrTables),
                            ctypes.POINTER(_cabi.CrState), ctypes.POINTER(vp)]
    L.hs_destroy.argtypes = [vp]
    L.hs_reset.argtypes = [vp, vp, vp]
    L.hs_step.argtypes = [vp, vp, vp, vp, vp]
    L.hs_render.argtypes = [vp, vp]
    L.hs_semantic.argtypes = [vp, vp]
    L.hs_simt_blocks.restype = ctypes.c_long
    L.hs_frame_order.argtypes = [vp, vp, vp]
    L.hs_last_error.restype = ctypes.c_char_p
    L.hs_geom.argtypes = [ctypes.POINTER(_cabi.CrConfig), vp]
    L.hs_geom_fields.restype = ctypes.c_char_p
    _libs[key] = L
  return _libs[key]


def config(num_envs=1, area=(64, 64), view=(9, 9), size=(64, 64), length=10000, reward=True, auto_reset=False,
           slot_capacity=None, n_daylight=None, seed=0, env_offset=0, item_size=(1, 1), digit_size=(1, 1)):
  """A cr_config (include/crafter_b200.h) as Env builds it, without the render tables: enough for the
  checks cr_create makes before it touches a buffer."""
  return _cabi.CrConfig(
      num_envs=num_envs, area_w=area[0], area_h=area[1], view_w=view[0], view_h=view[1], size_w=size[0],
      size_h=size[1], length=length, reward=int(reward), auto_reset=int(auto_reset),
      slot_capacity=slot_capacity or state_lib.default_slot_capacity(area),
      n_daylight=n_daylight or length + 1026, item_w=item_size[0], item_h=item_size[1], digit_w=digit_size[0],
      digit_h=digit_size[1], seed=seed, env_offset=env_offset)


def geom(area=(64, 64), view=(9, 9), size=(64, 64)):
  """{field: value} of what cr_create makes of a geometry (tests/simt hs_geom: the Geom fields the kernels
  branch on and the launch decisions at the H100's shared-memory limit); ValueError with the message
  cr_create fails with."""
  L = simt_lib()
  names = L.hs_geom_fields().decode().split(',')
  out = np.zeros(len(names), np.int64)
  cfg = config(area=area, view=view, size=size)
  if L.hs_geom(ctypes.byref(cfg), out.ctypes.data) != 0:
    raise ValueError(L.hs_last_error().decode())
  return dict(zip(names, (int(v) for v in out)))


class HostSimEnv:

  def __init__(self, num_envs=1, area=(64, 64), view=(9, 9), size=(64, 64), reward=True,
               length=10000, seed=0, auto_reset=False, env_offset=0, slot_capacity=None,
               max_obj_tiles=None, final_obs=False):
    self._L = self._load(max_obj_tiles)
    geo = tables_lib.geometry(view, size)
    self.B, self.area = num_envs, tuple(area)
    self.size = tuple(int(v) for v in geo['size'])
    self.capacity = slot_capacity or state_lib.default_slot_capacity(area)
    nc = area[0] * area[1]
    nch = -(-area[0] // 12) * -(-area[1] // 12)
    B = num_envs
    self.state = dict(
        mat=np.zeros((B, nc), np.uint8), objmap=np.zeros((B, nc), np.uint16),
        ents=np.zeros((B, self.capacity), np.int64), inventory=np.zeros((B, 16), np.int32),
        achievements=np.zeros((B, 22), np.int32), pstate=np.zeros((B, 16), np.int32),
        touched=np.zeros((B, (nch + 31) // 32), np.uint32), perm=np.zeros((B, 512), np.uint8),
        next_mat=np.zeros((B, nc), np.uint8), next_ents=np.zeros((B, self.capacity), np.int64),
        next_meta=np.zeros((B, 8), np.int32),
        reset_list=np.zeros(B, np.int32), reset_count=np.zeros(1, np.int32),
        ep_return=np.zeros((B, 2), np.float64), final_stats=np.zeros((B, 42), np.int32),
        balance_list=np.zeros(B, np.int32), balance_count=np.zeros(1, np.int32))
    if os.environ.get('CRAFTER_B200_INCR_CENSUS') != '0':
      self.state['chunk_cnt'] = np.zeros((B, nch * 2), np.int32)
    t = tables_lib.render_tables(tuple(int(v) for v in geo['view']), self.size)
    n_day = int(length) + 1026  # like crafter_b200.Env: slack for done envs that are stepped on
    self.tables = {k: np.ascontiguousarray(t[k]) for k in (
        'mat_tex', 'obj_tex', 'item_tile', 'vignette', 'colx', 'rowy')}
    self.tables['daylight'] = tables_lib.daylight_table(n_day)
    cfg = _cabi.CrConfig(
        num_envs=B, area_w=area[0], area_h=area[1], view_w=int(geo['view'][0]),
        view_h=int(geo['view'][1]), size_w=self.size[0], size_h=self.size[1], length=int(length),
        reward=int(reward), auto_reset=int(auto_reset), slot_capacity=self.capacity,
        n_daylight=n_day, item_w=t['item_size'][0], item_h=t['item_size'][1],
        digit_w=t['digit_size'][0], digit_h=t['digit_size'][1], seed=seed, env_offset=env_offset)
    tabs = _cabi.CrTables(**{k: v.ctypes.data for k, v in self.tables.items()})
    st = _cabi.CrState(**{k: v.ctypes.data for k, v in self.state.items()})
    self.final_obs = np.zeros((B, self.size[1], self.size[0], 3), np.uint8) if final_obs else None
    self.final_semantic = np.zeros((B,) + tuple(area), np.uint8) if final_obs else None
    if final_obs:
      st.final_obs = self.final_obs.ctypes.data
      st.final_semantic = self.final_semantic.ctypes.data
    self.h = ctypes.c_void_p()
    assert self._L.hs_create(ctypes.byref(cfg), ctypes.byref(tabs), ctypes.byref(st),
                           ctypes.byref(self.h)) == 0
    self.obs = np.zeros((B, self.size[1], self.size[0], 3), np.uint8)
    self.reward = np.zeros(B, np.float32)
    self.done = np.zeros(B, np.uint8)

  @staticmethod
  def _load(max_obj_tiles):
    return lib(max_obj_tiles)

  def reset(self, mask=None):
    m = None if mask is None else np.ascontiguousarray(mask, np.uint8)
    self._L.hs_reset(self.h, None if m is None else m.ctypes.data, self.obs.ctypes.data)
    return self.obs

  def step(self, actions):
    a = np.ascontiguousarray(actions, np.int32)
    self._L.hs_step(self.h, a.ctypes.data, self.obs.ctypes.data, self.reward.ctypes.data,
                  self.done.ctypes.data)
    return self.obs, self.reward, self.done.astype(bool)

  def render(self):
    self._L.hs_render(self.h, self.obs.ctypes.data)
    return self.obs

  def recount(self):
    """After writing state['mat'] directly: refresh what the implementation keeps about the terrain."""
    self._L.hs_recount.argtypes = [ctypes.c_void_p]
    self._L.hs_recount(self.h)

  def semantic(self):
    out = np.zeros((self.B,) + self.area, np.uint8)
    self._L.hs_semantic(self.h, out.ctypes.data)
    return out

  def set_inventory(self, values, env_ids=None):
    idx = slice(None) if env_ids is None else env_ids
    for name, amount in values.items():
      self.state['inventory'][idx, rules.ITEMS.index(name)] = amount
      if name == 'health':
        self.state['pstate'][idx, state_lib.PS['player_last_health']] = amount
        self.state['pstate'][idx, state_lib.PS['env_last_health']] = amount

  def snapshot(self, i):
    s = self.state
    return state_lib.canonical(s['mat'][i], s['ents'][i], s['inventory'][i], s['achievements'][i],
                               s['pstate'][i], s['touched'][i], self.area)


class SimtEnv(HostSimEnv):
  """The same numpy-driven env on tests/simt: the product's KERNELS (block / warp choreography
  included) on the SIMT emulator instead of the per-lane device functions of tests/hostsim."""

  @staticmethod
  def _load(max_obj_tiles):
    return simt_lib(max_obj_tiles)
