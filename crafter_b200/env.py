"""Batched Crafter environment on one H100: the `crafter.Env` surface (crafter/env.py:25-130) with a
`num_envs` batch dimension and torch.cuda tensors in and out.

Host code stays Python; all simulation and rendering runs in hand-written sm_90a kernels behind
the C ABI of include/crafter_b200.h.  torch is used for device memory and streams only.
"""
import collections
import ctypes
import os

import numpy as np
import torch

from . import _cabi
from . import rules
from . import state as state_lib
from . import tables as tables_lib

DiscreteSpace = collections.namedtuple('DiscreteSpace', 'n')  # env.py:18-21 (gym is optional)
BoxSpace = collections.namedtuple('BoxSpace', 'low, high, shape, dtype')
OBSERVATIONS = ('rgb', 'semantic', 'symbolic')
MAX_LEVEL = 2 ** 31 - 2  # the largest world seed of the reference, hash(...) % (2**31 - 1) (env.py:74)
LEVEL_SAMPLED = -2  # Env.levels of an env that draws its worlds from the level table (Env.sample_levels)
MAX_WEIGHT_TOTAL = 2 ** 32 - 1  # the largest total weight of a level table
# player.facing as (dx, dy) by the facing index of the player record (objects.py:33-34: left, right, up, down)
FACING = ((-1, 0), (1, 0), (0, -1), (0, 1))
# The 22 channels of every window cell of observation='symbolic' (layout: include/crafter_b200.h,
# cr_step_symbolic): one-hot of the material, set under objects too, then one-hot of the object's texture
SYMBOLIC_CHANNELS = tuple(rules.MATERIALS) + (
    'player', 'cow', 'zombie', 'skeleton', 'arrow-left', 'arrow-right', 'arrow-up', 'arrow-down', 'plant',
    'plant-ripe')


def symbolic_layout(grid):
  """{part: slice} of the symbolic vector of a local view `grid` = (gx, gy): 'map' (22 gx gy entries, cell
  (x, y) at (x * gy + y) * 22, channels SYMBOLIC_CHANNELS), 'inventory' (16, count / 9 in rules.ITEMS
  order), 'facing' (4, one-hot in FACING order), 'sleeping' (1) and 'daylight' (1)."""
  start, out = 0, {}
  for part, n in (('map', len(SYMBOLIC_CHANNELS) * grid[0] * grid[1]), ('inventory', len(rules.ITEMS)),
                  ('facing', len(FACING)), ('sleeping', 1), ('daylight', 1)):
    out[part] = slice(start, start + n)
    start += n
  return out


def player_facing(ents):
  """info['facing']: the player's facing (dx, dy) as int32 (B, 2), decoded from the `aux` field (bits 48-63)
  of the player's slot record (slot 1) in the ents tensor (B, slot_capacity) int64."""
  table = torch.tensor(FACING, dtype=torch.int32, device=ents.device)
  return table[(ents[:, 1] >> 48).long()]


def daylight_at(pstate, daylight):
  """info['daylight']: the daylight each env's last step used (env.py:135-139), float32 (B,): the daylight
  table at the env's step counter, clamped to the table's end as the kernels clamp it."""
  step = pstate[:, state_lib.PS['step']].long().clamp(0, daylight.numel() - 1)
  return daylight[step].float()


def check_levels(levels, mask, num_envs):
  """Env.set_levels' arguments checked on the host: (levels as int64, mask as bool or None), tensors on the
  device `levels` came on.  ValueError for a non-integer dtype, a wrong shape, or a masked entry that is
  neither -1 nor a world seed in [0, MAX_LEVEL]; entries outside the mask are not looked at."""
  if torch.is_tensor(levels):
    if levels.dtype.is_floating_point or levels.dtype.is_complex or levels.dtype == torch.bool:
      raise ValueError(f'levels must be integers, not {levels.dtype}')
    arr = levels.to(torch.int64)
  else:
    a = np.asarray(levels)
    if a.dtype.kind not in 'iu':
      raise ValueError(f'levels must be integers, not {a.dtype}')
    if a.dtype.kind == 'u' and a.size and int(a.max()) > MAX_LEVEL:
      raise ValueError(f'levels must be -1 or world seeds in [0, {MAX_LEVEL}]')
    arr = torch.from_numpy(a.astype(np.int64))
  if tuple(arr.shape) != (num_envs,):
    raise ValueError(f'levels must have shape ({num_envs},), not {tuple(arr.shape)}')
  if mask is not None:
    mask = torch.as_tensor(mask, device=arr.device).to(torch.bool)
    if tuple(mask.shape) != (num_envs,):
      raise ValueError(f'mask must have shape ({num_envs},), not {tuple(mask.shape)}')
  chosen = arr if mask is None else torch.where(mask, arr, -1)  # -1 is always valid
  lo, hi = torch.stack([chosen.min(), chosen.max()]).tolist() if num_envs else (-1, -1)  # one device read
  if lo < -1 or hi > MAX_LEVEL:
    raise ValueError(f'levels must be -1 or world seeds in [0, {MAX_LEVEL}]')
  return arr, mask


def _int_vector(values, name):
  """`values` as a 1-d int64 tensor (on the device it came on); ValueError for another dtype or shape."""
  if torch.is_tensor(values):
    if values.dtype.is_floating_point or values.dtype.is_complex or values.dtype == torch.bool:
      raise ValueError(f'{name} must be integers, not {values.dtype}')
    arr = values.to(torch.int64)
  else:
    a = np.asarray(values)
    if a.dtype.kind not in 'iu':
      raise ValueError(f'{name} must be integers, not {a.dtype}')
    if a.dtype.kind == 'u' and a.size and int(a.max()) > MAX_WEIGHT_TOTAL:
      raise ValueError(f'{name} out of range')
    arr = torch.from_numpy(a.astype(np.int64))
  if arr.dim() != 1:
    raise ValueError(f'{name} must have shape (n,), not {tuple(arr.shape)}')
  return arr


def check_level_weights(weights, n):
  """Level table weights checked on the host (one read when they are on a device): int64 (n,), non-negative
  integers whose total lies in [1, MAX_WEIGHT_TOTAL].  ValueError otherwise."""
  arr = _int_vector(weights, 'weights')
  if tuple(arr.shape) != (n,):
    raise ValueError(f'weights must have shape ({n},), not {tuple(arr.shape)}')
  lo, hi = torch.stack([arr.min(), arr.max()]).tolist()
  if lo < 0 or hi > MAX_WEIGHT_TOTAL:  # (a larger entry could wrap the int64 total around)
    raise ValueError(f'weights must be integers in [0, {MAX_WEIGHT_TOTAL}]')
  total = int(arr.sum())
  if not 1 <= total <= MAX_WEIGHT_TOTAL:
    raise ValueError(f'the total weight must lie in [1, {MAX_WEIGHT_TOTAL}], not {total}')
  return arr


def check_level_table(seeds, weights=None):
  """Env.set_level_table's arguments checked on the host: (seeds, weights) as int64 (n,) tensors, n >= 1.
  ValueError for a non-integer dtype, a wrong shape, a seed outside [0, MAX_LEVEL], a negative weight or a total
  weight outside [1, MAX_WEIGHT_TOTAL]; weights=None is weight 1 for every seed."""
  arr = _int_vector(seeds, 'seeds')
  n = arr.numel()
  if n < 1:
    raise ValueError('the level table needs at least one seed')
  lo, hi = torch.stack([arr.min(), arr.max()]).tolist()
  if lo < 0 or hi > MAX_LEVEL:
    raise ValueError(f'seeds must be world seeds in [0, {MAX_LEVEL}]')
  w = torch.ones(n, dtype=torch.int64) if weights is None else check_level_weights(weights, n)
  return arr, w


class Info(dict):
  """`info` of Env.step (env.py:108-115) as batched tensors; expensive entries are computed on
  first access: 'semantic' (engine.py:251-264), 'discount' (env.py:111) and -- for auto_reset, where
  'inventory' / 'achievements' of an env that just finished already belong to its next episode --
  'final_inventory' / 'final_achievements' / 'final_player_pos' / 'final_observation' / 'final_semantic': the terminal transition as the
  reference's info shows it (rows of envs with done=False hold their last terminal values or zeros).
  'world_seed' int32 (B,): the world seed the current episode of each env plays; 'final_world_seed' int32 (B,):
  the world seed of the episode that ended in this step (rows with done=False hold older values or zeros) --
  with auto_reset, what Env.reset(levels=...) needs to replay that episode (see Env.set_levels).

  What the frame shows beyond the semantic ids (a semantic window shows every player as id 13):
  'facing' int32 (B, 2), the player's facing (dx, dy); 'sleeping' bool (B,); 'daylight' float32 (B,), the
  daylight of the step.  'local_semantic': the local semantic window (see Env.local_semantic), which is
  `obs` itself with observation='semantic'."""

  def __init__(self, env, *args, **kwargs):
    super().__init__(*args, **kwargs)
    self._env = env

  def __missing__(self, key):
    env = self._env
    if key == 'semantic':
      value = env.semantic()
    elif key == 'discount':
      # env.py:111: 1 - float(dead).  Taken from the terminal record of the tick (a regenerated env's
      # inventory already shows the health of its next episode): dead is only ever set with done
      dead = env._done & (env._state['final_stats'][:, 23] != 0)
      value = 1.0 - dead.float()
    elif key == 'final_achievements':
      value = env._state['final_stats'][:, :22]
    elif key == 'final_inventory':
      value = env._state['final_stats'][:, 24:40]
    elif key == 'final_player_pos':
      value = env._state['final_stats'][:, 40:42]
    elif key in ('final_observation', 'final_semantic'):
      if env._final_semantic is None:
        raise KeyError(f"{key} needs Env(..., auto_reset=True, final_obs=True)")
      final = {'rgb': env._final_obs, 'semantic': env._final_local, 'symbolic': env._final_symbolic}[env._observation]
      value = final if key == 'final_observation' else env._final_semantic.view(env.num_envs, *env._area)
    elif key == 'facing':
      value = player_facing(env._state['ents'])
    elif key == 'sleeping':
      value = env._state['pstate'][:, state_lib.PS['sleeping']] != 0
    elif key == 'daylight':
      value = daylight_at(env._state['pstate'], env._daylight)
    elif key == 'world_seed':
      value = env._state['pstate'][:, state_lib.PS['world_seed']]
    elif key == 'final_world_seed':
      value = env._state['final_world_seed']
    elif key == 'local_semantic':
      value = env._local if env._observation == 'semantic' else env.local_semantic()
    else:
      raise KeyError(key)
    self[key] = value
    return value


class Env:
  """Drop-in for `crafter.Env(area, view, size, reward, length, seed)` (env.py:27-29) plus:

  num_envs      batch size; every tensor gains a leading dimension of this size
  device        a CUDA device (there is no CPU path)
  auto_reset    False (reference semantics: the caller resets, `reset(done)` takes a mask) or True:
                finished episodes are regenerated inside `step()` and the returned observation of
                those envs is the first one of the new episode
  env_offset    global index of env 0, so that a batch sharded over GPUs matches one big batch:
                env i plays the reference's `Env(seed=seed + env_offset + i)`
  final_obs     with auto_reset: also draw the frame of the step that ended an episode (the one the
                reference returns with done=True, env.py:96,118) into info['final_observation']
  observation   'rgb' (the reference's frames) or 'semantic': no frame is drawn inside the step, and obs is
                the local semantic window, uint8 (num_envs, gx, gy) with gx = view[0] and gy = view[1] minus
                the item rows, x-major like info['semantic']: the id of each cell the frame's local view
                shows (LocalView, engine.py:155-180; ids of SemanticView, engine.py:251-264: materials
                1..12, objects 13..18), 0 outside the map.  render() and info['semantic'] still work on
                demand; with final_obs, info['final_observation'] is the terminal window.  step_host is
                not available.
                Or 'symbolic': no frame either, and obs is float32 (num_envs, D), D = 22 gx gy + 22 (1408
                at the default view): the local window one-hot by material and by object texture, the
                inventory / 9, the facing one-hot, sleeping and the daylight.  The layout is defined in
                include/crafter_b200.h (cr_step_symbolic); decode it through SYMBOLIC_CHANNELS and
                Env.symbolic_layout rather than by offsets.  render(), info['semantic'] and
                local_semantic() work on demand; with final_obs, info['final_observation'] is the terminal
                vector.  step_host is not available.

  Randomness is counter-based (Philox keyed by the per-episode world seed, see DESIGN.md), so a
  batch is reproducible and independent of how it is sharded.  An episode is a function of its world seed
  and its actions: set_levels / reset(levels=...) choose the world seeds (fixed evaluation worlds, finite
  training sets, level-replay curricula, replaying a logged episode); set_level_table / sample_levels make envs
  draw the world of every new episode from a weighted table of world seeds inside the step, and
  set_level_weights updates the weights without a host read.  Returned tensors are views of the
  env's output buffers: they are overwritten by the next `step()` / `reset()`; clone to keep them.
  """

  def __init__(self, num_envs=1, area=(64, 64), view=(9, 9), size=(64, 64), reward=True,
               length=10000, seed=None, device=None, auto_reset=False, env_offset=0,
               slot_capacity=None, final_obs=False, observation='rgb'):
    if not torch.cuda.is_available():
      raise RuntimeError('crafter_b200 needs a CUDA device (sm_90a); there is no CPU fallback')
    self._lib = _cabi.load()
    self._device = torch.device('cuda', torch.cuda.current_device()) if device is None else (
        torch.device(device))
    if self._device.type != 'cuda':
      raise ValueError('device must be a CUDA device')
    if self._device.index is None:
      self._device = torch.device('cuda', torch.cuda.current_device())
    geo = tables_lib.geometry(view, size)
    self._num_envs = int(num_envs)
    self._area = (int(area[0]), int(area[1]))
    self._view = geo['view']
    self._size = geo['size']
    self._reward = reward
    self._length = length
    self._seed = int(np.random.randint(0, 2 ** 31 - 1) if seed is None else seed)  # env.py:32
    if not 0 <= self._seed + env_offset + num_envs < 2 ** 61 - 1:
      raise ValueError('seed out of range')
    self._auto_reset = bool(auto_reset)
    if final_obs and not auto_reset:
      raise ValueError('final_obs only makes sense with auto_reset=True (otherwise obs IS the terminal frame)')
    self._want_final_obs = bool(final_obs)
    if observation not in OBSERVATIONS:
      raise ValueError(f"observation must be one of {OBSERVATIONS}, not {observation!r}")
    self._observation = observation
    self._grid = tuple(int(v) for v in geo['grid'])  # the local view (env.py:42-44): the window's shape
    self._env_offset = int(env_offset)
    self._capacity = int(slot_capacity or state_lib.default_slot_capacity(self._area))
    # env.py:106: length None / 0 = no time limit.  Daylight (env.py:135-139) is a host-built table, so an
    # unbounded env gets a million steps of it (8 MB; a random agent lives 170); running past the table
    # keeps its last entry and raises the ERR_DAYLIGHT_CLAMP bit, which check_errors() reports
    # (a done env may be stepped on without a reset, as the reference allows: 1024 steps of slack)
    self._n_daylight = int(length) + 1026 if length else 1_000_002
    self.reward_range = None  # env.py:55-56
    self.metadata = None
    with torch.cuda.device(self._device):
      self._stream = torch.cuda.Stream(self._device)
      self._alloc_state()
      self._daylight = self._upload(tables_lib.daylight_table(self._n_daylight))
      self._handle, self._tables = self._create(tuple(int(v) for v in self._size))
    self._aux_handles = {}
    self._table, self._table_len = None, 0  # set_level_table
    self._needs_reset = True
    # raw addresses of the fixed buffers: the per-step calls below hand them to the C ABI without
    # touching torch again (the library switches to its own device itself, see DeviceGuard)
    self._ptrs = (self._actions.data_ptr(), self._out.data_ptr(), self._reward_buf.data_ptr(), self._done.data_ptr())
    self._step_fn = {'rgb': self._lib.cr_step, 'semantic': self._lib.cr_step_local,
                     'symbolic': self._lib.cr_step_symbolic}[observation]
    self._stream_ptr = self._stream.cuda_stream
    self._host_key, self._host_ptrs = None, None

  # ---- construction ---------------------------------------------------------------------------
  def _upload(self, array):
    return torch.from_numpy(np.ascontiguousarray(array)).to(self._device)

  def _alloc_state(self):
    B, nc = self._num_envs, self._area[0] * self._area[1]
    nch = -(-self._area[0] // 12) * -(-self._area[1] // 12)
    z = lambda *shape, dtype: torch.zeros(*shape, dtype=dtype, device=self._device)
    self._state = dict(
        mat=z(B, nc, dtype=torch.uint8),
        objmap=z(B, nc, dtype=torch.int16),
        ents=z(B, self._capacity, dtype=torch.int64),
        inventory=z(B, len(rules.ITEMS), dtype=torch.int32),
        achievements=z(B, len(rules.ACHIEVEMENTS), dtype=torch.int32),
        pstate=z(B, len(rules.PSTATE), dtype=torch.int32),
        touched=z(B, (nch + 31) // 32, dtype=torch.int32),
        perm=z(B, 512, dtype=torch.uint8),
        next_mat=z(B, nc, dtype=torch.uint8),
        next_ents=z(B, self._capacity, dtype=torch.int64),
        next_meta=z(B, 8, dtype=torch.int32),
        reset_list=z(B, dtype=torch.int32),
        ep_return=z(B, 2, dtype=torch.float64),
        final_stats=z(B, 42, dtype=torch.int32),
        balance_list=z(B, dtype=torch.int32),
        level=torch.full((B,), -1, dtype=torch.int32, device=self._device),  # set_levels
        final_world_seed=z(B, dtype=torch.int32))
    counters = z(4, dtype=torch.int32)  # adjacent, so the step graph clears both with one memset
    self._state['reset_count'] = counters[0:1]
    self._state['balance_count'] = counters[1:2]
    if os.environ.get('CRAFTER_B200_INCR_CENSUS') != '0':
      # grass / path cells per chunk, maintained by the terrain writes instead of being re-counted by
      # every balance tick (DESIGN.md 4.2; =0 goes back to the census for A/B runs)
      self._state['chunk_cnt'] = z(B, nch * 2, dtype=torch.int32)
    mode, want = self._observation, self._want_final_obs
    frame, dim = (int(self._size[1]), int(self._size[0]), 3), self.symbolic_layout['daylight'].stop
    self._obs = z(B, *frame, dtype=torch.uint8) if mode == 'rgb' else None
    self._local = z(B, *self._grid, dtype=torch.uint8) if mode == 'semantic' else None
    self._sym = z(B, dim, dtype=torch.float32) if mode == 'symbolic' else None
    self._out = {'rgb': self._obs, 'semantic': self._local, 'symbolic': self._sym}[mode]  # what step() returns
    self._final_obs = z(B, *frame, dtype=torch.uint8) if want and mode == 'rgb' else None
    self._final_local = z(B, *self._grid, dtype=torch.uint8) if want and mode == 'semantic' else None
    self._final_symbolic = z(B, dim, dtype=torch.float32) if want and mode == 'symbolic' else None
    self._final_semantic = z(B, nc, dtype=torch.uint8) if want else None
    self._reward_buf = z(B, dtype=torch.float32)
    self._zero_reward = z(B, dtype=torch.float32)  # reward=False (env.py:116-117); info['reward'] keeps the real one
    self._done = z(B, dtype=torch.bool)
    self._actions = z(B, dtype=torch.int32)
    self._level_in = z(B, dtype=torch.int32)  # set_levels' argument on the device
    self._level_mask = z(B, dtype=torch.uint8)

  def _create(self, size):
    t = tables_lib.render_tables(tuple(int(v) for v in self._view), size)
    dev = {k: self._upload(t[k]) for k in ('mat_tex', 'obj_tex', 'item_tile', 'vignette', 'colx',
                                           'rowy')}
    dev['daylight'] = self._daylight
    cfg = _cabi.CrConfig(
        num_envs=self._num_envs, area_w=self._area[0], area_h=self._area[1],
        view_w=int(self._view[0]), view_h=int(self._view[1]), size_w=size[0], size_h=size[1],
        length=int(self._length or 0), reward=int(bool(self._reward)),
        auto_reset=int(self._auto_reset), slot_capacity=self._capacity,
        n_daylight=self._n_daylight, item_w=t['item_size'][0], item_h=t['item_size'][1],
        digit_w=t['digit_size'][0], digit_h=t['digit_size'][1], seed=self._seed,
        env_offset=self._env_offset)
    tabs = _cabi.CrTables(**{k: v.data_ptr() for k, v in dev.items()})
    st = _cabi.CrState(**{k: v.data_ptr() for k, v in self._state.items()})
    if self._final_semantic is not None and size == tuple(int(v) for v in self._size):
      if self._final_obs is not None:
        st.final_obs = self._final_obs.data_ptr()
      elif self._final_local is not None:
        st.final_local = self._final_local.data_ptr()
      else:
        st.final_symbolic = self._final_symbolic.data_ptr()
      st.final_semantic = self._final_semantic.data_ptr()
    handle = ctypes.c_void_p()
    _cabi.check(self._lib.cr_create(
        ctypes.byref(cfg), ctypes.byref(tabs), ctypes.byref(st), ctypes.byref(handle)))
    return handle, dev

  def close(self):
    for h, _ in list(getattr(self, '_aux_handles', {}).values()) + [
        (getattr(self, '_handle', None), None)]:
      if h:
        self._lib.cr_destroy(h)
    self._aux_handles = {}
    self._handle = None

  def __del__(self):
    try:
      self.close()
    except Exception:
      pass

  # ---- spaces (env.py:58-68) ------------------------------------------------------------------
  @property
  def num_envs(self):
    return self._num_envs

  @property
  def device(self):
    return self._device

  @property
  def observation(self):
    """'rgb', 'semantic' or 'symbolic' (see the class docstring)."""
    return self._observation

  @property
  def symbolic_layout(self):
    """{part: slice} of the symbolic vector at this env's view (see symbolic_layout())."""
    return symbolic_layout(self._grid)

  @property
  def observation_space(self):
    if self._observation == 'semantic':
      return BoxSpace(0, 18, self._grid, np.uint8)
    if self._observation == 'symbolic':
      return BoxSpace(0, 1, (self.symbolic_layout['daylight'].stop,), np.float32)
    return BoxSpace(0, 255, (int(self._size[1]), int(self._size[0]), 3), np.uint8)

  @property
  def action_space(self):
    return DiscreteSpace(len(rules.ACTIONS))

  @property
  def action_names(self):
    return rules.ACTIONS

  # ---- stream plumbing ------------------------------------------------------------------------
  def _enter(self):
    self._stream.wait_stream(torch.cuda.current_stream(self._device))
    return self._stream.cuda_stream

  def _exit(self):
    torch.cuda.current_stream(self._device).wait_stream(self._stream)

  # ---- Env.reset (env.py:70-81) ---------------------------------------------------------------
  def reset(self, mask=None, levels=None):
    """Start a new episode in every env (or in those where `mask` is True); returns obs.  With `levels`, this
    is set_levels(levels, mask) followed by the reset: the episodes it starts play those levels."""
    with torch.cuda.device(self._device):
      ptr = None
      if mask is not None:
        mask = torch.as_tensor(mask, device=self._device).to(torch.bool).contiguous()
        assert mask.shape == (self._num_envs,)
        if self._needs_reset and not bool(mask.all()):
          raise RuntimeError('the first reset() must cover every env (envs outside the mask have no world yet)')
        ptr = mask.data_ptr()
      if levels is not None:
        self.set_levels(levels, mask)
      s = self._enter()
      if self._observation == 'semantic':  # no frame: the windows of the state the reset left
        _cabi.check(self._lib.cr_reset(self._handle, ptr, None, s))
        _cabi.check(self._lib.cr_local(self._handle, self._local.data_ptr(), s))
      elif self._observation == 'symbolic':  # no frame: the vectors of the state the reset left
        _cabi.check(self._lib.cr_reset(self._handle, ptr, None, s))
        _cabi.check(self._lib.cr_symbolic(self._handle, self._sym.data_ptr(), s))
      else:
        _cabi.check(self._lib.cr_reset(self._handle, ptr, self._obs.data_ptr(), s))
      self._exit()
    self._needs_reset = False
    return self._out

  # ---- levels ---------------------------------------------------------------------------------
  def set_levels(self, levels, mask=None):
    """Choose the world of each env's next episodes (semantics: include/crafter_b200.h, cr_set_levels).

    levels  int tensor / array of shape (num_envs,): -1 = the reference's sequence (episode e of env i plays
            world seed hash((seed + env_offset + i, e)) % (2**31 - 1)), or a world seed s in [0, 2**31 - 2]:
            every episode of that env that starts from now on plays world s, exactly the reference's
            World.reset(seed=s) + generate_world, until the level changes again (auto-reset replays it).
    mask    bool (num_envs,) or None (all): entries of `levels` outside the mask are ignored.

    The running episodes are left alone; the last assignment before an episode starts wins.  With auto_reset,
    call it at any time and the new level takes effect from each env's next episode (its world is generated
    once, now); reset(mask, levels) right after a step starts the new level at once, at the price of
    generating the worlds of those envs twice in that step.  Checked on the host (ValueError) before anything
    is launched."""
    arr, mask = check_levels(levels, mask, self._num_envs)  # (also takes the masked envs out of sampling)
    with torch.cuda.device(self._device):
      arr = arr.to(self._device)
      if mask is not None:
        mask = mask.to(self._device)
      self._level_in.copy_(arr if mask is None else torch.where(mask, arr, -1))
      if mask is not None:
        self._level_mask.copy_(mask)
      s = self._enter()
      _cabi.check(self._lib.cr_set_levels(self._handle, None if mask is None else self._level_mask.data_ptr(),
                                          self._level_in.data_ptr(), s))
      self._exit()

  @property
  def levels(self):
    """A copy of the current level of every env, int32 (num_envs,) (-1: the reference's sequence, -2 =
    LEVEL_SAMPLED: drawn from the level table, see sample_levels)."""
    return self._state['level'].clone()

  # ---- the level sampler ------------------------------------------------------------------------
  def set_level_table(self, seeds, weights=None):
    """The table the sampled envs (sample_levels) draw their worlds from (semantics: include/crafter_b200.h,
    cr_set_level_table): `seeds` (n,) ints in [0, MAX_LEVEL], `weights` (n,) non-negative ints (None: all 1)
    whose total lies in [1, 2**32 - 1]; a seed of weight 0 is never drawn.  Every new episode of a sampled env
    draws one seed with probability weight / total, inside the step: no world is generated twice and the
    host is not read.  The draw is keyed by (seed + env_offset + env, episode), so a run replays from the
    seed and the table contents, however the batch is sharded.

    Checked on the host (ValueError); this is the rare call.  Replacing the table later is allowed at any
    time, with the staleness described under set_level_weights."""
    seeds, weights = check_level_table(seeds, weights)
    n = seeds.numel()
    with torch.cuda.device(self._device):
      if self._table is None or n > self._table['seeds'].numel():  # the buffers belong to the env; grown, never shrunk
        z = lambda *shape, dtype: torch.zeros(*shape, dtype=dtype, device=self._device)
        table = dict(seeds=z(n, dtype=torch.int32), cum=z(n, dtype=torch.int32), n=z(1, dtype=torch.int32),
                     weights=z(n, dtype=torch.int64))
        _cabi.check(self._lib.cr_set_level_table(self._handle, table['seeds'].data_ptr(), table['cum'].data_ptr(),
                                                 table['n'].data_ptr(), n))
        self._table = table
      self._table_len = n
      self._table['n'].fill_(n)
      self._table['seeds'][:n].copy_(seeds)
      self._write_weights(weights.to(self._device), n)

  def _write_weights(self, weights, n):
    """int64 device weights (n,) -> the kept copy and the inclusive cumulative sum as uint32 bit patterns."""
    self._table['weights'][:n].copy_(weights)
    cum = torch.cumsum(weights, 0)  # int64: exact
    self._table['cum'][:n].copy_(cum.view(torch.int32)[0::2])  # the low words (little-endian)

  def set_level_weights(self, weights):
    """New weights for the seeds of the level table, (n,) non-negative ints: the per-step call of a
    prioritized-level-replay loop.  A device tensor is only checked for dtype and shape and is not read
    back: nothing here synchronises, and keeping the total in [1, 2**32 - 1] is the caller's part (a zero
    total makes the sampled envs play the reference's sequence and raises an error bit that check_errors()
    reports; a larger total wraps around).  Host arrays are checked like set_level_table's.  Float
    priorities p in [0, 1] are meant to come in as `(p * 2**24).round().to(torch.int64)`, which keeps the
    total of up to 255 levels in range; scale down for more.

    Nothing in flight is touched: each env's prefetched next world and the seed prepared for the one after it
    were drawn from the table as it stood and are played as drawn, so new weights reach an env from its third
    new episode at the latest -- the price of never generating a world twice.  sample_levels(mask) makes
    them hold from the very next episode of the masked envs, at the cost of generating those worlds again.
    Weights need not be rewritten every step: a curriculum that updates them every few steps pays less."""
    if self._table is None:
      raise RuntimeError('set_level_weights: no level table (call set_level_table first)')
    n = self._table_len
    if torch.is_tensor(weights) and weights.is_cuda:
      arr = _int_vector(weights, 'weights')
      if tuple(arr.shape) != (n,):
        raise ValueError(f'weights must have shape ({n},), not {tuple(arr.shape)}')
    else:
      arr = check_level_weights(weights, n)
    with torch.cuda.device(self._device):
      self._write_weights(arr.to(self._device), n)

  def sample_levels(self, mask=None):
    """The envs where `mask` is True (None: all) draw the world of every new episode from the level table
    (set_level_table), until set_levels puts them on a level (or -1) again; `levels` shows LEVEL_SAMPLED = -2
    for them.  Like set_levels it leaves the running episodes alone and generates the next world of those
    envs once, now, from the table as it stands; reset(mask) right after it starts such episodes at once."""
    if self._table is None:
      raise RuntimeError('sample_levels: no level table (call set_level_table first)')
    with torch.cuda.device(self._device):
      if mask is not None:
        mask = torch.as_tensor(mask, device=self._device).to(torch.bool)
        if tuple(mask.shape) != (self._num_envs,):
          raise ValueError(f'mask must have shape ({self._num_envs},), not {tuple(mask.shape)}')
        self._level_mask.copy_(mask)
      s = self._enter()
      _cabi.check(self._lib.cr_sample_levels(self._handle, None if mask is None else self._level_mask.data_ptr(), s))
      self._exit()

  @property
  def level_table(self):
    """(seeds int32 (n,), weights int64 (n,)) copies of the level table, or None."""
    if self._table is None:
      return None
    n = self._table_len
    return self._table['seeds'][:n].clone(), self._table['weights'][:n].clone()

  # ---- Env.step (env.py:83-118) ---------------------------------------------------------------
  def step(self, actions):
    """actions: int tensor / array of shape (num_envs,) -> (obs, reward, done, info)."""
    if self._needs_reset:
      raise RuntimeError('call reset() before step()')  # the reference fails on None state too
    if not (torch.is_tensor(actions) and actions.data_ptr() == self._ptrs[0]):
      a = torch.as_tensor(actions)
      self._actions.copy_(a.reshape(self._num_envs), non_blocking=True)
    s = self._enter()
    _cabi.check(self._step_fn(self._handle, *self._ptrs, s))
    self._exit()
    info = Info(
        self, inventory=self._state['inventory'], achievements=self._state['achievements'],
        player_pos=self._state['pstate'][:, 12:14], reward=self._reward_buf)
    return self._out, self._reward_buf if self._reward else self._zero_reward, self._done, info

  @property
  def actions_buffer(self):
    """Write actions here and pass this very tensor to step() to skip the copy."""
    return self._actions

  def step_host(self, actions_pinned, reward_pinned, done_pinned, obs_pinned=None):
    """One tick through `cr_step_host`: pinned host buffers in and out, copies and the stream
    synchronisation included -- the path a non-torch caller of the reference's step() binds."""
    if self._observation != 'rgb':
      raise RuntimeError(f'step_host draws frames: it is not available with observation={self._observation!r}')
    if self._needs_reset:
      raise RuntimeError('call reset() before step()')
    key = (id(actions_pinned), id(reward_pinned), id(done_pinned), id(obs_pinned))
    if key != self._host_key:  # same buffers every step in a rollout loop: look the addresses up once
      self._host_ptrs = (actions_pinned.data_ptr(), obs_pinned.data_ptr() if obs_pinned is not None else None,
                         reward_pinned.data_ptr(), done_pinned.data_ptr())
      self._host_key, self._host_keep = key, (actions_pinned, reward_pinned, done_pinned, obs_pinned)
    _cabi.check(self._lib.cr_step_host(self._handle, *self._host_ptrs, *self._ptrs, self._stream_ptr))

  # ---- Env.render (env.py:120-130) ------------------------------------------------------------
  def render(self, size=None, env_ids=None):
    """Fresh (num_envs, H, W, 3) uint8 render, at `size` if given (e.g. 512 for videos); with
    `env_ids` only those envs are drawn, in that order: (len(env_ids), H, W, 3)."""
    with torch.cuda.device(self._device):
      if size is None:
        handle, sz = self._handle, tuple(int(v) for v in self._size)
      else:
        sz = tuple(size) if hasattr(size, '__len__') else (int(size), int(size))
        if sz not in self._aux_handles:
          self._aux_handles[sz] = self._create(sz)
        handle = self._aux_handles[sz][0]
      if env_ids is None:
        out = torch.empty(self._num_envs, sz[1], sz[0], 3, dtype=torch.uint8, device=self._device)
        s = self._enter()
        _cabi.check(self._lib.cr_render(handle, out.data_ptr(), s))
      else:
        ids = torch.as_tensor(env_ids, dtype=torch.int64).reshape(-1)
        if ids.numel() and (int(ids.min()) < 0 or int(ids.max()) >= self._num_envs):
          raise IndexError('env_ids out of range')
        ids = ids.to(device=self._device, dtype=torch.int32)
        out = torch.empty(ids.numel(), sz[1], sz[0], 3, dtype=torch.uint8, device=self._device)
        s = self._enter()
        _cabi.check(self._lib.cr_render_envs(handle, ids.data_ptr(), ids.numel(), out.data_ptr(), s))
      self._exit()
    return out

  def semantic(self):
    """info['semantic'] (engine.py:251-264): (num_envs, W, H) uint8."""
    with torch.cuda.device(self._device):
      out = torch.empty(self._num_envs, *self._area, dtype=torch.uint8, device=self._device)
      s = self._enter()
      _cabi.check(self._lib.cr_semantic(self._handle, out.data_ptr(), s))
      self._exit()
    return out

  def local_semantic(self):
    """The local semantic window of every env as the state stands: (num_envs, gx, gy) uint8, the obs of
    observation='semantic' (see the class docstring).  Reads only the cells around each player."""
    with torch.cuda.device(self._device):
      out = torch.empty(self._num_envs, *self._grid, dtype=torch.uint8, device=self._device)
      s = self._enter()
      _cabi.check(self._lib.cr_local(self._handle, out.data_ptr(), s))
      self._exit()
    return out

  def symbolic(self):
    """The symbolic vector of every env as the state stands: (num_envs, D) float32, the obs of
    observation='symbolic' (see the class docstring), in any mode."""
    with torch.cuda.device(self._device):
      out = torch.empty(self._num_envs, self.symbolic_layout['daylight'].stop, dtype=torch.float32,
                        device=self._device)
      s = self._enter()
      _cabi.check(self._lib.cr_symbolic(self._handle, out.data_ptr(), s))
      self._exit()
    return out

  # ---- inspection -----------------------------------------------------------------------------
  @property
  def state(self):
    """The raw SoA state tensors (zero copy); layout in csrc/cr_common.h."""
    return self._state

  @property
  def launch_count(self):
    return int(self._lib.cr_launch_count(self._handle))

  def error_flags(self):
    """OR of the envs' sticky error bits (synchronises): 1 = an object was dropped because the slot
    arena was full (raise slot_capacity), 2 = an env was stepped past its daylight table, 4 = a sampled env
    was seeded from an empty level table (no table, or a total weight of 0)."""
    flags = ctypes.c_int32(0)
    s = self._enter()
    _cabi.check(self._lib.cr_error_flags(self._handle, ctypes.byref(flags), s))
    self._exit()
    return int(flags.value)

  def check_errors(self):
    """Raise if any env has a sticky error bit set (see error_flags)."""
    flags = self.error_flags()
    if flags & 1:
      bad = self._state['pstate'][:, 14].bitwise_and(1).nonzero().flatten().tolist()
      raise RuntimeError(f'crafter_b200: slot arena overflow in envs {bad[:8]}{"..." if len(bad) > 8 else ""}: an object '
                         f'was dropped (slot_capacity={self._capacity}); results of those envs differ from the reference')
    if flags & 2:
      raise RuntimeError('crafter_b200: an env was stepped past its daylight table '
                         f'({self._n_daylight} entries); daylight is frozen at the last entry there')
    if flags & 4:
      raise RuntimeError('crafter_b200: a sampled env was seeded from an empty level table (total weight 0, or '
                         'no table); it played the world of the reference sequence instead')

  def set_inventory(self, values, env_ids=None):
    """Overwrite inventory entries ({item: amount}), like poking `env._player.inventory` on the
    reference.  Health also resets the two `_last_health` trackers (env.py:77, objects.py:78)."""
    inv, ps = self._state['inventory'], self._state['pstate']
    idx = slice(None) if env_ids is None else torch.as_tensor(env_ids, device=self._device)
    for name, amount in values.items():
      inv[idx, rules.ITEMS.index(name)] = int(amount)
      if name == 'health':
        ps[idx, state_lib.PS['player_last_health']] = int(amount)
        ps[idx, state_lib.PS['env_last_health']] = int(amount)

  def snapshot(self, i):
    """Canonical host copy of env i's state (see state.canonical)."""
    torch.cuda.synchronize(self._device)
    g = lambda k: self._state[k][i].cpu().numpy()
    return state_lib.canonical(g('mat'), g('ents'), g('inventory'), g('achievements'), g('pstate'),
                               g('touched'), self._area)

  def state_dict(self):
    torch.cuda.synchronize(self._device)
    return {k: v.clone() for k, v in self._state.items()}

  def load_state_dict(self, sd):
    # snapshots taken before levels existed: every env on the reference's sequence
    sd = dict(sd)
    if 'level' not in sd and 'final_world_seed' not in sd:
      sd['level'] = torch.full_like(self._state['level'], -1)
      sd['final_world_seed'] = torch.zeros_like(self._state['final_world_seed'])
    if set(sd) != set(self._state):
      raise ValueError(f'state_dict of another layout (keys differ: {sorted(set(sd) ^ set(self._state))})')
    torch.cuda.synchronize(self._device)
    for k, v in self._state.items():
      v.copy_(sd[k])
    self._needs_reset = False

  def recount(self):
    """After writing `state['mat']` directly: refresh what the library keeps incrementally about the
    terrain (the per-chunk grass / path counts; CRAFTER_B200_INCR_CENSUS=0 keeps nothing)."""
    s = self._enter()
    _cabi.check(self._lib.cr_recount(self._handle, s))
    self._exit()
