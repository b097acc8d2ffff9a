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
LEVEL_PINNED_BASE = -3  # Env.levels of an env pinned to table entry e is LEVEL_PINNED_BASE - e (Env.pin_levels)
# cr_author_levels' status bits (include/crafter_b200.h): why a world was rejected
AUTHOR_REASONS = ((1, 'a byte out of range (material outside 1..12 or creature outside 0..3)'),
                  (2, 'a creature on a cell that is not grass, sand or path'),
                  (4, 'the start cell (W/2, H/2) is not grass, sand or path, or holds a creature'),
                  (8, 'more than slot_capacity - 2 creatures'),
                  (16, 'the entry lies outside the cache, or appears twice in the call'))
# cr_mutate_levels' status bit beyond AUTHOR_REASONS: why a child was rejected
MUTATE_REASONS = AUTHOR_REASONS + (
    (32, 'the parent lies outside the cache, or its row does not hold its current world'),)
# cr_mutate_levels' edit kinds, in op order: set a material (rules.MATERIALS), place a creature, remove a creature
MUTATE_OPS = tuple(rules.MATERIALS) + ('cow', 'zombie', 'skeleton', 'remove')
MAX_MUTATE_EDITS = 4096  # CR_MUTATE_MAX_EDITS
MAX_WEIGHT_TOTAL = 2 ** 32 - 1  # the largest total weight of a level table
# the columns of a level statistics row (include/crafter_b200.h, cr_set_level_stats); 5.. are the achievements
START_WORDS = 20  # CR_START_WORDS: a level start record is on, x, y, facing, then the 16 items (Env.set_level_starts)
FACING_NAMES = ('left', 'right', 'up', 'down')  # the facing index of a start record (FACING order)
ERR_LEVEL_START = 8  # error_flags: a level start was on but not applicable; that episode started at the reference's
LEVEL_STATS = ('episodes', 'terminated', 'length', 'return_tenths', 'return_tenths_sq')
LEVEL_STATS_COLUMNS = len(LEVEL_STATS) + len(rules.ACHIEVEMENTS)
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


def pack_worlds(materials, creatures, area):
  """Env.author_levels' worlds: materials (k, W, H) ids 1..12 and creatures (k, W, H) 0..3 (None: none), integer
  tensors or arrays, as the uint8 (k, W * H) bytes of cr_author_levels (x-major, material | creature << 4), on the
  device `materials` came on.  ValueError for a non-integer dtype or a wrong shape; a value out of range becomes
  the byte 0xC0, which cr_author_levels rejects with status bit 1."""
  def as_tensor(values, name):
    if not torch.is_tensor(values):
      values = np.asarray(values)
      if values.dtype.kind not in 'iu':
        raise ValueError(f'{name} must be integers, not {values.dtype}')
      values = torch.from_numpy(values.astype(np.int64))
    elif values.dtype.is_floating_point or values.dtype.is_complex or values.dtype == torch.bool:
      raise ValueError(f'{name} must be integers, not {values.dtype}')
    if values.dim() != 3 or tuple(values.shape[1:]) != tuple(area):
      raise ValueError(f'{name} must have shape (k, {area[0]}, {area[1]}), not {tuple(values.shape)}')
    return values.to(torch.int64)
  mat = as_tensor(materials, 'materials')
  cre = torch.zeros_like(mat) if creatures is None else as_tensor(creatures, 'creatures').to(mat.device)
  if cre.shape != mat.shape:
    raise ValueError(f'creatures must have the shape of materials, {tuple(mat.shape)}, not {tuple(cre.shape)}')
  ok = (mat >= 1) & (mat <= 12) & (cre >= 0) & (cre <= 3)
  return torch.where(ok, mat | (cre << 4), 0xC0).to(torch.uint8).reshape(mat.shape[0], -1)


def mutate_weights(weights):
  """Env.mutate_levels' weights as a list of MUTATE_OPS ints: None (every op 1), a sequence of 16 ints in op order,
  or a dict {op name: weight} (missing ops: 0).  ValueError for an unknown name, a wrong length, a non-integer or
  negative weight, or a total outside [1, MAX_WEIGHT_TOTAL]."""
  if weights is None:
    return [1] * len(MUTATE_OPS)
  if isinstance(weights, dict):
    unknown = set(weights) - set(MUTATE_OPS)
    if unknown:
      raise ValueError(f'unknown mutation ops {sorted(map(str, unknown))} (one of MUTATE_OPS)')
    weights = [weights.get(name, 0) for name in MUTATE_OPS]
  a = np.asarray(weights.cpu() if torch.is_tensor(weights) else weights)
  if a.dtype.kind not in 'iu' or a.shape != (len(MUTATE_OPS),):
    raise ValueError(f'weights must be {len(MUTATE_OPS)} integers (MUTATE_OPS order) or a dict, not {a.dtype} {a.shape}')
  w = [int(v) for v in a]
  if min(w) < 0:
    raise ValueError('mutation weights must be non-negative')
  if not 1 <= sum(w) <= MAX_WEIGHT_TOTAL:
    raise ValueError(f'the total mutation weight must lie in [1, {MAX_WEIGHT_TOTAL}], not {sum(w)}')
  return w


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


def goal_mask(names):
  """The level goal mask (Env.set_level_goals) of `names`: an achievement name, a sequence of names, or an int mask
  over the 22 achievements (bit k = rules.ACHIEVEMENTS[k]).  ValueError for an unknown name or a bit above 21."""
  if isinstance(names, str):
    names = (names,)
  if isinstance(names, (int, np.integer)) and not isinstance(names, (bool, np.bool_)):
    mask = int(names)
    if not 0 <= mask < 1 << len(rules.ACHIEVEMENTS):
      raise ValueError(f'a goal mask must lie in [0, 2**{len(rules.ACHIEVEMENTS)}), not {mask}')
    return mask
  mask = 0
  for name in names:
    if not isinstance(name, str) or name not in rules.ACHIEVEMENTS:
      raise ValueError(f'unknown achievement {name!r} (one of rules.ACHIEVEMENTS)')
    mask |= 1 << rules.ACHIEVEMENTS.index(name)
  return mask


def level_start(inventory=None, pos=None, facing='down', area=(64, 64)):
  """One level start record (Env.set_level_starts): int32 (20,) with `on` = 1.

  inventory  {item name: amount} (rules.ITEMS); items it leaves out take the reference's initial values (data.yaml:
             9 health, food, drink and energy, nothing else).  Every amount lies in [0, 9], health in [1, 9].
  pos        (x, y) inside `area`, or None: the reference's start (W/2, H/2).
  facing     'left', 'right', 'up', 'down', or a (dx, dy) pair of FACING.
  ValueError for an unknown name, a value out of range or a position outside the area.  Whether the world's cell can
  hold the player (grass, sand or path, no creature) is decided on the device, when the episode is installed."""
  W, H = (int(v) for v in area)
  row = np.zeros(START_WORDS, np.int32)
  row[0] = 1
  x, y = (W // 2, H // 2) if pos is None else pos
  if not (isinstance(x, (int, np.integer)) and isinstance(y, (int, np.integer)) and 0 <= x < W and 0 <= y < H):
    raise ValueError(f'a start position must be integers (x, y) inside the area {W} x {H}, not {pos!r}')
  row[1:3] = x, y
  if isinstance(facing, str):
    if facing not in FACING_NAMES:
      raise ValueError(f'unknown facing {facing!r} (one of {FACING_NAMES})')
    row[3] = FACING_NAMES.index(facing)
  else:
    try:
      row[3] = FACING.index(tuple(int(v) for v in facing))
    except (TypeError, ValueError):
      raise ValueError(f'a facing is a name of {FACING_NAMES} or a (dx, dy) of {FACING}, not {facing!r}') from None
  inv = [rules.ITEM_INITIAL.get(name, 0) for name in rules.ITEMS]
  for name, amount in (inventory or {}).items():
    if name not in rules.ITEMS:
      raise ValueError(f'unknown item {name!r} (one of rules.ITEMS)')
    if not isinstance(amount, (int, np.integer)) or isinstance(amount, (bool, np.bool_)):
      raise ValueError(f'the amount of {name} must be an int, not {amount!r}')
    inv[rules.ITEMS.index(name)] = int(amount)
  row[4:] = inv
  _check_starts(row[None], area)
  return row


def _check_starts(rows, area):
  """Start records (k, 20) int64 checked on the host: on in {0, 1}; the records that are on lie inside `area`, face
  one of the four directions, and hold items in [0, 9] with health in [1, 9].  ValueError naming the first bad row."""
  rows = np.asarray(rows, np.int64)
  W, H = area
  on = rows[:, 0] != 0
  inv = rows[:, 4:]
  bad = (rows[:, 0] < 0) | (rows[:, 0] > 1) | on & (
      (rows[:, 1] < 0) | (rows[:, 1] >= W) | (rows[:, 2] < 0) | (rows[:, 2] >= H) | (rows[:, 3] < 0) |
      (rows[:, 3] > 3) | (inv < 0).any(1) | (inv > rules.ITEM_MAX).any(1) | (inv[:, 0] < 1))
  if bad.any():
    i = int(np.flatnonzero(bad)[0])
    raise ValueError(f'start {i} is not a level start record (on 0 or 1; x, y inside {W} x {H}; facing 0..3; items '
                     f'in [0, 9], health in [1, 9]): {rows[i].tolist()}')


def level_scores(stats):
  """(percent float64 (n, 22), score float64 (n,)) of Env.level_stats() rows, on their device: the success rate of
  every achievement in percent of the entry's episodes (rules.ACHIEVEMENTS order) and the Crafter score, the
  geometric mean with an offset of 1%, exp(mean(log(1 + percent))) - 1, as the reference's analysis computes them
  (analysis/common.py:36, 47-55).  NaN for entries without episodes."""
  episodes = stats['episodes'].to(torch.float64)
  percent = 100 * stats['achievements'].to(torch.float64) / episodes[:, None]  # 0 / 0 = NaN
  return percent, torch.exp(torch.log(1 + percent).mean(1)) - 1


class Info(dict):
  """`info` of Env.step (env.py:108-115) as batched tensors; expensive entries are computed on
  first access: 'semantic' (engine.py:251-264), 'discount' (env.py:111) and -- for auto_reset, where
  'inventory' / 'achievements' of an env that just finished already belong to its next episode --
  'final_inventory' / 'final_achievements' / 'final_player_pos' / 'final_observation' / 'final_semantic': the terminal transition as the
  reference's info shows it (rows of envs with done=False hold their last terminal values or zeros).
  'world_seed' int32 (B,): the world seed the current episode of each env plays; 'final_world_seed' int32 (B,):
  the world seed of the episode that ended in this step (rows with done=False hold older values or zeros) --
  with auto_reset, what Env.reset(levels=...) needs to replay that episode (see Env.set_levels).
  With a level table: 'level_entry' int32 (B,), the table entry the current episode of each env was drawn from or
  pinned to (-1: none); 'final_level_entry' int32 (B,), the entry of the episode that ended in this step (rows with
  done=False hold older values or -1) -- what a learner-side level score is attributed by (see Env.level_stats).
  'goal' int32 (B,): the level goal mask of the current episode of each env (0: the reference's reward; see
  Env.set_level_goals); 'final_goal' int32 (B,): the goal of the episode that ended in this step, 0 in rows with
  done=False.

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
      # inventory already shows the health of its next episode): dead is only ever set with done.  Its flag is
      # 1 * dead | 2 * reached (set_level_goals): a reached goal ends the task too, with discount 0
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
    elif key in ('level_entry', 'final_level_entry'):
      if env._ring is None:
        raise KeyError(f'{key} needs a level table (Env.set_level_table)')
      if key == 'final_level_entry':
        value = env._ring['final']
      else:
        episode = env._state['pstate'][:, state_lib.PS['episode']].long() & 3
        value = env._ring['entry'].gather(1, episode[:, None])[:, 0]
    elif key in ('goal', 'final_goal'):
      if env._goals is None:
        value = torch.zeros(env.num_envs, dtype=torch.int32, device=env._device)
      else:
        episode = env._state['pstate'][:, state_lib.PS['episode']].long()
        if key == 'final_goal':  # with auto_reset the episode that ended is the one before; its slot is still intact
          episode = episode - int(env._auto_reset)
        value = env._goals['notes'].gather(1, (episode & 3)[:, None])[:, 0]
        if key == 'final_goal':
          value = torch.where(env._done, value, 0)
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
  set_level_weights updates the weights without a host read; author_levels puts caller-made worlds into table
  entries and pin_levels puts envs on one entry; set_level_stats / level_stats count every finished episode
  against the entry it was drawn from, for the caller's level scores; set_level_goals gives entries achievement
  goals that pay the reward and end the episode, and set_level_starts the player's start position, facing,
  inventory and vitals.  Returned tensors are views of the
  env's output buffers: they are overwritten by the next `step()` / `reset()`; clone to keep them.

  Streams (the contract: include/crafter_b200.h, "Streams and ordering"): every call is ordered behind the work
  queued on the caller's current stream of the env's device and leaves its results ready for that stream, so
  writes to inputs or state and reads of earlier outputs need no synchronisation as long as they run on it.
  Host actions (numpy, lists, pinned or pageable CPU tensors) are read before step() returns; step_host
  synchronises.  One env belongs to one thread at a time.  Capturing step() into the caller's own CUDA graph
  is not supported.
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
    self._cache = None  # set_level_cache
    self._ring = None  # the entry notes of cr_set_level_stats, registered with the level table
    self._stats = None  # set_level_stats
    self._goals = None  # set_level_goals: the goal table and the notes
    self._starts = None  # set_level_starts: the start table and the notes
    self._needs_reset = True
    # raw addresses of the fixed buffers: the per-step calls below hand them to the C ABI without
    # touching torch again (the library switches to its own device itself, see DeviceGuard)
    self._ptrs = (self._actions.data_ptr(), self._out.data_ptr(), self._reward_buf.data_ptr(), self._done.data_ptr())
    self._step_fn = {'rgb': self._lib.cr_step, 'semantic': self._lib.cr_step_local,
                     'symbolic': self._lib.cr_step_symbolic}[observation]
    self._stream_ptr = self._stream.cuda_stream
    self._entered = torch.cuda.Event()  # _enter()
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
  # Every entry point that launches work calls _enter() and runs on the stream it returns, so that work is
  # ordered behind everything the caller queued before the call (the contract: include/crafter_b200.h, "Streams
  # and ordering"); tests/test_env_streams.py checks that no entry point passes another stream to the library.
  def _enter(self):
    current = torch.cuda.current_stream(self._device)
    if not current.query():  # (an idle stream has nothing left to wait for: step_host's loop pays no event)
      self._entered.record(current)  # one event, recorded again by every call
      self._stream.wait_event(self._entered)
    return self._stream_ptr

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
    LEVEL_SAMPLED: drawn from the level table, see sample_levels; LEVEL_PINNED_BASE - e = -3 - e: pinned to table
    entry e, see pin_levels)."""
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
      if self._cache is not None:  # new rows for a grown table; only the rows whose seed changed are generated
        self._fill_level_cache()
      if self._ring is None or (self._stats is not None and self._stats.shape[0] < self._table['seeds'].numel()):
        self._register_level_stats(self._stats is not None)
      if self._goals is not None and self._goals['goals'].numel() < self._table['seeds'].numel():
        self._register_level_goals()
      if self._starts is not None and self._starts['starts'].shape[0] < self._table['seeds'].numel():
        self._register_level_starts()

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

  # ---- the level cache ------------------------------------------------------------------------------
  def set_level_cache(self, enabled=True):
    """Keep the world of every level table entry generated on the device, so that sampled envs copy their next
    world instead of generating it (semantics: include/crafter_b200.h, cr_set_level_cache).  Every output and
    the state stay bit-identical to a run without the cache; only time and memory change.

    enabled=True allocates one row per entry of the table's buffers and generates the worlds, on the caller's
    stream; later set_level_table calls generate only the rows whose seed changed (and add rows when the table
    grows); set_level_weights never touches the cache.  enabled=False frees the rows.  The memory is
    level_cache['bytes']: about 6.2 KB per world at area 64 x 64 (slot capacity 256), about 96 KB at 256 x 256;
    a table of 2**20 seeds at the default geometry takes about 6.5 GB.  Envs on level -1 or a fixed level are
    not cached."""
    if not enabled:
      if self._cache is not None:
        _cabi.check(self._lib.cr_set_level_cache(self._handle, None, None, None, None, None, 0))
        self._cache = None
      return
    if self._table is None:
      raise RuntimeError('set_level_cache: no level table (call set_level_table first)')
    with torch.cuda.device(self._device):
      self._fill_level_cache()

  def _fill_level_cache(self):
    """(Re)register rows for every entry of the table's buffers, grown with the table (the rows held so far are
    kept), and generate the worlds of the entries in use whose row does not hold their seed."""
    rows = self._table['seeds'].numel()
    old = self._cache
    if old is None or old['tag'].numel() < rows:
      z = lambda *shape, dtype: torch.zeros(*shape, dtype=dtype, device=self._device)
      cache = dict(mat=z(rows, self._area[0] * self._area[1], dtype=torch.uint8),
                   ents=z(rows, self._capacity, dtype=torch.int64), meta=z(rows, 2, dtype=torch.int32),
                   tag=torch.full((rows,), -1, dtype=torch.int32, device=self._device),
                   row=old['row'] if old else torch.full((self._num_envs, 2), -1, dtype=torch.int32, device=self._device))
      if old is not None:  # (the last fill ran on the env's stream, which _exit() made this stream wait for)
        for k in ('mat', 'ents', 'meta', 'tag'):
          cache[k][:old[k].shape[0]].copy_(old[k])
      for v in cache.values():  # read by the env's stream: not reused by torch before that stream is done
        v.record_stream(self._stream)
      _cabi.check(self._lib.cr_set_level_cache(self._handle, *(cache[k].data_ptr() for k in (
          'mat', 'ents', 'meta', 'tag', 'row')), rows))
      self._cache = cache
    s = self._enter()
    _cabi.check(self._lib.cr_fill_level_cache(self._handle, 0, self._table_len, s))
    self._exit()

  @property
  def level_cache(self):
    """None without a level cache, else {'rows': worlds it can hold, 'bytes_per_world', 'bytes': all of it}
    (set_level_cache states the sizes)."""
    if self._cache is None:
      return None
    c = self._cache
    rows = c['tag'].numel()
    per_world = sum(c[k].element_size() * c[k][0].numel() for k in ('mat', 'ents', 'meta', 'tag'))
    return dict(rows=rows, bytes_per_world=per_world,
                bytes=per_world * rows + c['row'].element_size() * c['row'].numel())

  # ---- per-level episode statistics ------------------------------------------------------------------
  def _register_level_stats(self, with_stats):
    """Register the entry notes (allocated once, sized by the batch: filled with -1) and, with_stats, one statistics
    row per row of the table's buffers, grown with the table (the rows counted so far are kept)."""
    B = self._num_envs
    if self._ring is None:
      self._ring = dict(entry=torch.full((B, 4), -1, dtype=torch.int32, device=self._device),
                        final=torch.full((B,), -1, dtype=torch.int32, device=self._device))
      for v in self._ring.values():  # written by the env's stream: not reused by torch before that stream is done
        v.record_stream(self._stream)
    stats, rows = None, 0
    if with_stats:
      rows = self._table['seeds'].numel()
      stats = self._stats
      if stats is None or stats.shape[0] < rows:
        stats = torch.zeros(rows, LEVEL_STATS_COLUMNS, dtype=torch.int64, device=self._device)
        if self._stats is not None:  # (the last step ran on the env's stream, which _exit() made this stream wait for)
          stats[:self._stats.shape[0]].copy_(self._stats)
        stats.record_stream(self._stream)
    _cabi.check(self._lib.cr_set_level_stats(self._handle, self._ring['entry'].data_ptr(), self._ring['final'].data_ptr(),
                                             None if stats is None else stats.data_ptr(), rows))
    self._stats = stats

  def set_level_stats(self, enabled=True):
    """Count every finished episode against the level table entry it was drawn from or pinned to (semantics:
    include/crafter_b200.h, cr_set_level_stats): per entry, the episodes, the terminated ones, the summed length,
    the summed return and its square in tenths (exact integers), and per achievement the episodes that unlocked it.
    The step only adds integers, so the counts are exact, reproducible and the same however the batch is sharded;
    level_stats() reads them and level_scores() or any torch code turns them into weights for set_level_weights,
    without a host read.

    enabled=True allocates one row per row of the table's buffers (216 bytes each), zeroed; the rows grow with the
    table and keep their counts.  enabled=False frees them.  An episode counts when it ends while the statistics
    are on; its entry was noted when its seed was decided, so an env moved off the table mid-episode still counts
    that episode under the entry it was drawn from.  A done report counts once per step that reports it: without
    auto_reset, stepping a done env again counts it again.  reset() of a running episode counts nothing.  Level -1
    and fixed-level episodes are not counted."""
    if not enabled:
      if self._stats is not None:
        self._register_level_stats(False)
      return
    if self._table is None:
      raise RuntimeError('set_level_stats: no level table (call set_level_table first)')
    with torch.cuda.device(self._device):
      if self._stats is None:
        self._register_level_stats(True)

  def level_stats(self):
    """Copies of the statistics rows of the n entries in use, made on the caller's stream (no host read):
    {'episodes', 'terminated', 'length', 'return_tenths', 'return_tenths_sq': int64 (n,), 'achievements': int64
    (n, 22) in rules.ACHIEVEMENTS order}.  The mean return of entry i is return_tenths[i] / (10 * episodes[i])."""
    if self._stats is None:
      raise RuntimeError('level_stats: the level statistics are off (call set_level_stats first)')
    with torch.cuda.device(self._device):
      rows = self._stats[:self._table_len]
      out = {k: rows[:, i].clone(memory_format=torch.contiguous_format) for i, k in enumerate(LEVEL_STATS)}
      out['achievements'] = rows[:, len(LEVEL_STATS):].clone(memory_format=torch.contiguous_format)
    return out

  def clear_level_stats(self, entries=None):
    """Zero the statistics rows of `entries` in [0, n) (None: all), ordered on the caller's stream like every call:
    how a caller keeps a window of recent episodes.  Checked on the host (ValueError; one read of device entries)."""
    if self._stats is None:
      raise RuntimeError('clear_level_stats: the level statistics are off (call set_level_stats first)')
    with torch.cuda.device(self._device):
      if entries is None:
        self._stats.zero_()
        return
      arr = self._entries(entries, 'clear_level_stats')
      self._check_entries(arr)
      self._stats[arr.to(self._device)] = 0

  # ---- level goals -----------------------------------------------------------------------------------
  def _register_level_goals(self):
    """Register the goal table, one entry per row of the table's buffers, grown with the table (the goals set so far
    are kept, new entries are 0), and the notes (allocated once, sized by the batch: filled with 0)."""
    rows = self._table['seeds'].numel()
    old = self._goals
    goals = torch.zeros(rows, dtype=torch.int32, device=self._device)
    notes = torch.zeros(self._num_envs, 4, dtype=torch.int32, device=self._device) if old is None else old['notes']
    if old is not None:  # (the last step ran on the env's stream, which _exit() made this stream wait for)
      goals[:old['goals'].numel()].copy_(old['goals'])
    for v in (goals, notes):  # read and written by the env's stream: not reused by torch before that stream is done
      v.record_stream(self._stream)
    _cabi.check(self._lib.cr_set_level_goals(self._handle, goals.data_ptr(), notes.data_ptr(), rows))
    self._goals = dict(goals=goals, notes=notes)

  def set_level_goals(self, goals):
    """Give level table entries goals (semantics: include/crafter_b200.h, cr_set_level_goals): an episode drawn from
    or pinned to entry i with goal G != 0 pays 1.0 in the step that first unlocks every achievement of G, and nothing
    else (no health term), and that step ends it (done; final_stats' flag 2, so info['discount'] is 0 and
    VectorEnv's `terminated` is True).  G = 0 is the reference's reward and ending.  So a (world, goal) pair is one
    table entry, and sample_levels, set_level_weights, pin_levels, the level cache and level_stats work on tasks as
    they do on worlds; a goal entry's successes are level_stats()['return_tenths'] / 10.

    goals  (n,) ints, one achievement mask per table entry (bit k = rules.ACHIEVEMENTS[k]; see goal_mask), or a
           list of n items that are each an achievement name, a sequence of names or an int; or None: no goals.
    A device int tensor is only checked for dtype and shape and is not read back (nothing synchronises; bits 22..31
    are ignored); host input is checked (ValueError for an unknown name or a bit above 21).

    An episode's goal is fixed when its world seed is decided, so a rewritten goal has the staleness of rewritten
    weights: it reaches an env from its third new episode at the latest, and from the next one after
    sample_levels / pin_levels.  The goal table grows with the level table (new entries: 0).  Level -1 and
    fixed-level episodes have no goal."""
    if goals is None:
      if self._goals is not None:
        _cabi.check(self._lib.cr_set_level_goals(self._handle, None, None, 0))
        self._goals = None
      return
    if self._table is None:
      raise RuntimeError('set_level_goals: no level table (call set_level_table first)')
    n = self._table_len
    if torch.is_tensor(goals) and goals.is_cuda:
      arr = _int_vector(goals, 'goals')
    elif torch.is_tensor(goals) or isinstance(goals, np.ndarray):
      arr = _int_vector(goals, 'goals')
      bad = (arr < 0) | (arr >= 1 << len(rules.ACHIEVEMENTS))
      if bool(bad.any()):
        raise ValueError(f'goals must be masks in [0, 2**{len(rules.ACHIEVEMENTS)}) (entry {int(bad.nonzero()[0, 0])})')
    else:
      arr = torch.tensor([goal_mask(g) for g in goals], dtype=torch.int64)
    if tuple(arr.shape) != (n,):
      raise ValueError(f'goals must have shape ({n},), not {tuple(arr.shape)}')
    with torch.cuda.device(self._device):
      if self._goals is None:
        self._register_level_goals()
      self._goals['goals'][:n].copy_(arr.to(self._device))

  @property
  def level_goals(self):
    """A copy of the goal masks of the n table entries in use, int32 (n,), or None without goals."""
    if self._goals is None:
      return None
    return self._goals['goals'][:self._table_len].clone()

  # ---- level starts ------------------------------------------------------------------------------------
  def _register_level_starts(self):
    """Register the start table, one record per row of the table's buffers, grown with the table (the starts set so
    far are kept, new entries are 0), and the notes (allocated once, sized by the batch: filled with 0)."""
    rows = self._table['seeds'].numel()
    old = self._starts
    starts = torch.zeros(rows, START_WORDS, dtype=torch.int32, device=self._device)
    notes = (torch.zeros(self._num_envs, 4, START_WORDS, dtype=torch.int32, device=self._device)
             if old is None else old['notes'])
    if old is not None:  # (the last step ran on the env's stream, which _exit() made this stream wait for)
      starts[:old['starts'].shape[0]].copy_(old['starts'])
    for v in (starts, notes):  # read and written by the env's stream: not reused by torch before that stream is done
      v.record_stream(self._stream)
    _cabi.check(self._lib.cr_set_level_starts(self._handle, starts.data_ptr(), notes.data_ptr(), rows))
    self._starts = dict(starts=starts, notes=notes)

  def set_level_starts(self, starts):
    """Give level table entries player starts (semantics: include/crafter_b200.h, cr_set_level_starts): an episode
    drawn from or pinned to entry i whose record is on starts with the player at the record's (x, y), facing its
    way, with its inventory (health, food, drink and energy included) and both last healths at its health; nothing
    else about the fresh episode changes, and the world is still the one generated or authored for a start at the
    centre.  A record that is off (all zeros) is the reference's start.  So a task curriculum can start deep goals
    with their prerequisites (a stone pickaxe for collect_iron), and a probe is an authored world, a pinned env and a
    start.

    starts  (n, 20) ints, one record per table entry (see level_start), or a list of n items that are each None (the
            reference's start), a dict of level_start keyword arguments (area: this env's), or a record; or None: no
            starts.
    A device int tensor is only checked for dtype and shape and is not read back (nothing synchronises); the device
    decides whether a record is applicable when it installs an episode: the cell (x, y) must be grass, sand or path
    and hold no creature, the rest as level_start checks it.  A record that is on but not applicable starts that
    episode at the reference's start and raises error bit 8 (error_flags, check_errors).  Host input is checked
    (ValueError).

    An episode's start is fixed when its world seed is decided, like its goal: a rewritten start reaches an env from
    its third new episode at the latest, and from the next one after sample_levels / pin_levels.  The start table
    grows with the level table (new entries: 0).  Level -1 and fixed-level episodes start at the reference's start."""
    if starts is None:
      if self._starts is not None:
        _cabi.check(self._lib.cr_set_level_starts(self._handle, None, None, 0))
        self._starts = None
      return
    if self._table is None:
      raise RuntimeError('set_level_starts: no level table (call set_level_table first)')
    n = self._table_len
    if torch.is_tensor(starts) or isinstance(starts, np.ndarray):
      dtype = starts.dtype
      if (dtype.is_floating_point or dtype.is_complex or dtype == torch.bool) if torch.is_tensor(starts) else (
          dtype.kind not in 'iu'):
        raise ValueError(f'starts must be integers, not {dtype}')
      arr = starts.to(torch.int64) if torch.is_tensor(starts) else torch.from_numpy(starts.astype(np.int64))
      if not arr.is_cuda:
        if tuple(arr.shape) == (n, START_WORDS):
          _check_starts(arr.numpy(), self._area)
    else:
      rows = []
      for i, item in enumerate(starts):
        if item is None:
          rows.append(np.zeros(START_WORDS, np.int64))
        elif isinstance(item, dict):
          rows.append(level_start(**dict(dict(area=self._area), **item)))
        else:
          row = np.asarray(item)
          if row.dtype.kind not in 'iu' or row.shape != (START_WORDS,):
            raise ValueError(f'start {i} must be None, a dict of level_start arguments or {START_WORDS} ints')
          rows.append(row)
      arr = torch.from_numpy(np.array(rows, np.int64).reshape(-1, START_WORDS))
      _check_starts(arr.numpy(), self._area)
    if tuple(arr.shape) != (n, START_WORDS):
      raise ValueError(f'starts must have shape ({n}, {START_WORDS}), not {tuple(arr.shape)}')
    with torch.cuda.device(self._device):
      if self._starts is None:
        self._register_level_starts()
      self._starts['starts'][:n].copy_(arr.to(self._device))

  @property
  def level_starts(self):
    """A copy of the start records of the n table entries in use, int32 (n, 20), or None without starts."""
    if self._starts is None:
      return None
    return self._starts['starts'][:self._table_len].clone()

  # ---- authored levels and pinning ----------------------------------------------------------------
  def _entries(self, entries, name, count=None):
    """`entries` as int64 (k,) on the host-checked range [0, n) of the level table (one read)."""
    if self._table is None:
      raise RuntimeError(f'{name}: no level table (call set_level_table first)')
    arr = _int_vector(entries, 'entries')
    if count is not None and arr.numel() != count:
      raise ValueError(f'entries must have shape ({count},), not {tuple(arr.shape)}')
    return arr

  def _check_entries(self, arr):
    n = self._table_len
    if arr.numel():
      lo, hi = torch.stack([arr.min(), arr.max()]).tolist()
      if lo < 0 or hi >= n:
        raise ValueError(f'entries must be level table entries in [0, {n})')

  def author_levels(self, entries, materials, creatures=None):
    """Write caller-made worlds into the level table's entries (semantics: include/crafter_b200.h,
    cr_author_levels): materials (k, W, H) ids 1..12 (the info['semantic'] ids), creatures (k, W, H) 0 none,
    1 cow, 2 zombie, 3 skeleton (None: none), for the k entries of `entries` in [0, n).  An episode on an
    authored entry i plays that world with every later draw keyed by seeds[i] and reports seeds[i] as its
    world seed; the player starts at (W/2, H/2) as in every episode, so that cell must be grass, sand or path
    without a creature, and creatures may stand on grass, sand and path only.  Sampled envs draw the entry
    with its weight, and pin_levels plays it in every episode.

    Turns the level cache on if it is off (the worlds live in its rows).  All or nothing: when any world is
    rejected, ValueError names the worlds and the reasons and no entry changes.  Reads a status word per world
    back, one synchronisation: this is the rare call.  An authored entry stays authored while its seed stays;
    set_level_table with another seed for it generates that seed's world over it.  Reaches the envs that
    already drew or were pinned to the entry from their second new episode at the latest; pin_levels or
    sample_levels again makes it hold from the next."""
    arr = self._entries(entries, 'author_levels')
    worlds = pack_worlds(materials, creatures, self._area)
    if worlds.shape[0] != arr.numel():
      raise ValueError(f'{arr.numel()} entries for {worlds.shape[0]} worlds')
    self._check_entries(arr)
    with torch.cuda.device(self._device):
      if self._cache is None:
        self._fill_level_cache()
      k = arr.numel()
      if k == 0:
        return
      ent = arr.to(self._device, torch.int32)
      worlds = worlds.to(self._device)
      status = torch.empty(k, dtype=torch.int32, device=self._device)
      s = self._enter()
      _cabi.check(self._lib.cr_author_levels(self._handle, ent.data_ptr(), worlds.data_ptr(), k, status.data_ptr(), s))
      self._exit()
      status = status.cpu().numpy()
    bad = np.flatnonzero(status)
    if len(bad):
      lines = [f'world {i} (entry {int(arr[i])}): ' + '; '.join(why for bit, why in AUTHOR_REASONS if status[i] & bit)
               for i in bad[:8]]
      more = f' (and {len(bad) - 8} more)' if len(bad) > 8 else ''
      raise ValueError(f'author_levels: {len(bad)} of {k} worlds rejected, nothing changed{more}:\n' + '\n'.join(lines))

  def level_worlds(self, entries):
    """The worlds the level cache holds for `entries` (k,) in [0, n), decoded from its rows: {'materials': uint8
    (k, W, H), 'creatures': uint8 (k, W, H) in author_levels' encoding, 'authored': bool (k,)}.  The read side of
    an edit loop: read, change in torch, author_levels.  A generated row shows its world as generation left it,
    so authoring it again under the same seed plays the same episodes."""
    if self._cache is None:
      raise RuntimeError('level_worlds: no level cache (call set_level_cache or author_levels first)')
    arr = self._entries(entries, 'level_worlds')
    self._check_entries(arr)
    W, H = self._area
    with torch.cuda.device(self._device):
      idx = arr.to(self._device)
      c, k = self._cache, arr.numel()
      materials = (c['mat'][idx] & 0x0F).reshape(k, W, H)
      ents = c['ents'][idx]
      n = c['meta'][idx, 0].to(torch.int64)
      kind = ents & 0xFF
      slot = torch.arange(self._capacity, device=self._device)
      live = (slot >= 2) & (slot < n[:, None]) & (kind >= 2) & (kind <= 4)
      x, y = (ents >> 16) & 0xFFFF, (ents >> 32) & 0xFFFF
      creatures = torch.zeros(k, W * H, dtype=torch.uint8, device=self._device)
      world = torch.arange(k, device=self._device)[:, None].expand_as(ents)
      creatures[world[live], (x * H + y)[live]] = (kind - 1)[live].to(torch.uint8)
      authored = (c['meta'][idx, 1] & 4) != 0
    return dict(materials=materials.contiguous(), creatures=creatures.reshape(k, W, H), authored=authored)

  def mutate_levels(self, parents, children, edits, key, weights=None):
    """Make children of level table entries on the device (semantics: include/crafter_b200.h, cr_mutate_levels):
    child i starts as the world the cache holds for parents[i], takes `edits` keyed random edits and is authored
    into entry children[i] (the mutator of ACCEL).  An edit sets a material, places a creature or removes one
    (MUTATE_OPS); edits keep the world valid, so a child of a valid world is never rejected for its bytes.  A child
    is a function of (parent world, key, child entry, edits, weights): the same call on every rank makes the same
    children, and a caller varies `key` between calls.

    parents, children  (k,) ints in [0, n); children distinct; a child may be its own parent or another's parent.
    edits              int in [0, MAX_MUTATE_EDITS].
    key                int in [0, 2**32).
    weights            None (every op 1), 16 ints in MUTATE_OPS order, or a dict {op name: weight}.
    Checked on the host (ValueError; one read of device entries).  Turns the level cache on if it is off.  A parent
    whose row does not hold its entry's current world (a seed rewritten without a fill) is rejected.  All or nothing,
    as author_levels: ValueError names the rejected children and the reasons, and no entry changes.  Reads a status
    word per child back, one synchronisation.  The children's statistics and goals are left alone.

    Returns {'materials': uint8 (k, W, H), 'creatures': uint8 (k, W, H)}: the children, as author_levels takes
    them."""
    arr_p = self._entries(parents, 'mutate_levels')
    arr_c = self._entries(children, 'mutate_levels', arr_p.numel())
    if isinstance(edits, bool) or not isinstance(edits, (int, np.integer)) or not 0 <= edits <= MAX_MUTATE_EDITS:
      raise ValueError(f'edits must be an int in [0, {MAX_MUTATE_EDITS}], not {edits!r}')
    if isinstance(key, bool) or not isinstance(key, (int, np.integer)) or not 0 <= key < 2 ** 32:
      raise ValueError(f'key must be an int in [0, 2**32), not {key!r}')
    w = mutate_weights(weights)
    k, n = arr_p.numel(), self._table_len
    if k:
      both = torch.cat([arr_p, arr_c.to(arr_p.device)])
      srt = torch.sort(arr_c).values
      dup = (srt[1:] == srt[:-1]).any() if k > 1 else torch.zeros((), dtype=torch.bool)
      lo, hi, twice = torch.stack([both.min(), both.max(), dup.to(both.device, torch.int64)]).tolist()  # one read
      if lo < 0 or hi >= n:
        raise ValueError(f'entries must be level table entries in [0, {n})')
      if twice:
        raise ValueError('children must be distinct')
    W, H = self._area
    with torch.cuda.device(self._device):
      if self._cache is None:
        self._fill_level_cache()
      if k == 0:
        empty = torch.zeros(0, W, H, dtype=torch.uint8, device=self._device)
        return dict(materials=empty, creatures=empty.clone())
      par = arr_p.to(self._device, torch.int32)
      chi = arr_c.to(self._device, torch.int32)
      worlds = torch.empty(k, W * H, dtype=torch.uint8, device=self._device)
      status = torch.empty(k, dtype=torch.int32, device=self._device)
      host_w = (ctypes.c_uint32 * len(MUTATE_OPS))(*w)
      s = self._enter()
      _cabi.check(self._lib.cr_mutate_levels(self._handle, par.data_ptr(), chi.data_ptr(), k, int(edits), host_w,
                                             int(key), worlds.data_ptr(), status.data_ptr(), s))
      self._exit()
      status = status.cpu().numpy()
    bad = np.flatnonzero(status)
    if len(bad):
      lines = [f'child {i} (entry {int(arr_c[i])}, parent {int(arr_p[i])}): ' +
               '; '.join(why for bit, why in MUTATE_REASONS if status[i] & bit) for i in bad[:8]]
      more = f' (and {len(bad) - 8} more)' if len(bad) > 8 else ''
      raise ValueError(f'mutate_levels: {len(bad)} of {k} children rejected, nothing changed{more}:\n' + '\n'.join(lines))
    worlds = worlds.reshape(k, W, H)
    return dict(materials=worlds & 0x0F, creatures=worlds >> 4)

  def pin_levels(self, entries, mask=None):
    """Pin each env where `mask` is True (None: all) to level table entry entries[env] in [0, n): every new
    episode of it plays that entry -- its seed, and its cached world (generated or authored) when the cache
    holds it -- whatever the weights, so an entry of weight 0 can serve as an evaluation level that sampled envs
    never draw.  `levels` shows LEVEL_PINNED_BASE - e.  Like set_levels it leaves the running episodes alone and
    builds the next world of those envs once, now; reset(mask) right after it starts them at once.  Checked on
    the host (ValueError; one read of device entries)."""
    arr = self._entries(entries, 'pin_levels', self._num_envs)
    with torch.cuda.device(self._device):
      if mask is not None:
        mask = torch.as_tensor(mask, device=self._device).to(torch.bool)
        if tuple(mask.shape) != (self._num_envs,):
          raise ValueError(f'mask must have shape ({self._num_envs},), not {tuple(mask.shape)}')
      arr = arr.to(self._device)
      self._check_entries(arr if mask is None else arr[mask])
      self._level_in.copy_(arr if mask is None else torch.where(mask, arr, 0))
      if mask is not None:
        self._level_mask.copy_(mask)
      s = self._enter()
      _cabi.check(self._lib.cr_pin_levels(self._handle, None if mask is None else self._level_mask.data_ptr(),
                                          self._level_in.data_ptr(), s))
      self._exit()

  # ---- Env.step (env.py:83-118) ---------------------------------------------------------------
  def step(self, actions):
    """actions: int tensor / array of shape (num_envs,) -> (obs, reward, done, info)."""
    if self._needs_reset:
      raise RuntimeError('call reset() before step()')  # the reference fails on None state too
    if not (torch.is_tensor(actions) and actions.data_ptr() == self._ptrs[0]):
      a = torch.as_tensor(actions).reshape(self._num_envs)
      if a.device.type == 'cpu':
        # Host actions are read before step() returns: the caller may refill its buffer at once.  They are
        # staged in a block of torch's pinned host cache, which is not handed out again before the copy has run.
        staged = torch.empty(self._num_envs, dtype=torch.int32, pin_memory=True)
        a = staged.copy_(a)
      self._actions.copy_(a, non_blocking=True)
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
    # behind the caller's queued work like every entry point; the call synchronises its stream, so nothing is
    # left for the caller's stream to wait on afterwards
    _cabi.check(self._lib.cr_step_host(self._handle, *self._host_ptrs, *self._ptrs, self._enter()))

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
    was seeded from an empty level table (no table, or a total weight of 0), 8 = an episode's level start was on but
    not applicable (its cell not grass, sand or path, or holding a creature; see set_level_starts) and the episode
    started at the reference's start."""
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
    if flags & ERR_LEVEL_START:
      bad = self._state['pstate'][:, 14].bitwise_and(ERR_LEVEL_START).nonzero().flatten().tolist()
      raise RuntimeError(f'crafter_b200: a level start was not applicable in envs {bad[:8]}{"..." if len(bad) > 8 else ""} '
                         '(its cell is not grass, sand or path, or holds a creature, or the record is out of range); '
                         "those episodes started at the reference's start")

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

  def state_dict(self, level_entries=False):
    """Copies of the state tensors.  level_entries=True (with a level table) adds 'level_entry', the entry notes of
    the running and the next two episodes (num_envs, 4), and 'final_level_entry', so that a restored batch counts
    its running episodes under the entries they were drawn from (set_level_stats).  They are opt-in so that
    snapshots of batches with and without a level table keep the same keys.  The level table, cache and statistics
    are not env state.  With level goals it adds 'level_goal', the goal notes (num_envs, 4), so that the running
    episodes keep their goals; the goal table itself is not env state either.  With level starts it adds
    'level_start', the start notes (num_envs, 4, 20), so that the episodes already decided keep their starts."""
    torch.cuda.synchronize(self._device)
    sd = {k: v.clone() for k, v in self._state.items()}
    if level_entries and self._ring is not None:
      sd['level_entry'], sd['final_level_entry'] = self._ring['entry'].clone(), self._ring['final'].clone()
    if level_entries and self._goals is not None:
      sd['level_goal'] = self._goals['notes'].clone()
    if level_entries and self._starts is not None:
      sd['level_start'] = self._starts['notes'].clone()
    return sd

  def load_state_dict(self, sd):
    # snapshots taken before levels existed: every env on the reference's sequence
    sd = dict(sd)
    if 'level' not in sd and 'final_world_seed' not in sd:
      sd['level'] = torch.full_like(self._state['level'], -1)
      sd['final_world_seed'] = torch.zeros_like(self._state['final_world_seed'])
    ring = {k: sd.pop(key) for k, key in (('entry', 'level_entry'), ('final', 'final_level_entry')) if key in sd}
    notes = sd.pop('level_goal', None)
    start_notes = sd.pop('level_start', None)
    if set(sd) != set(self._state):
      raise ValueError(f'state_dict of another layout (keys differ: {sorted(set(sd) ^ set(self._state))})')
    torch.cuda.synchronize(self._device)
    for k, v in self._state.items():
      v.copy_(sd[k])
    if ring and self._ring is None:
      self._register_level_stats(False)
    if self._ring is not None:  # snapshots without entry notes: no episode of theirs is attributed to an entry
      for k, v in self._ring.items():
        if k in ring:
          v.copy_(ring[k])
        else:
          v.fill_(-1)
    if notes is not None and self._goals is None:  # goal notes into a batch without goals: a goal table of zeros
      self.set_level_goals(torch.zeros(self._table_len, dtype=torch.int32, device=self._device))
    if self._goals is not None:  # snapshots without goal notes: their running episodes have no goal
      if notes is not None:
        self._goals['notes'].copy_(notes)
      else:
        self._goals['notes'].fill_(0)
    if start_notes is not None and self._starts is None:  # start notes into a batch without starts: a table of zeros
      self.set_level_starts(torch.zeros(self._table_len, START_WORDS, dtype=torch.int32, device=self._device))
    if self._starts is not None:  # snapshots without start notes: their decided episodes start at the reference's
      if start_notes is not None:
        self._starts['notes'].copy_(start_notes)
      else:
        self._starts['notes'].fill_(0)
    self._needs_reset = False

  def recount(self):
    """After writing `state['mat']` directly: refresh what the library keeps incrementally about the
    terrain (the per-chunk grass / path counts; CRAFTER_B200_INCR_CENSUS=0 keeps nothing)."""
    s = self._enter()
    _cabi.check(self._lib.cr_recount(self._handle, s))
    self._exit()
