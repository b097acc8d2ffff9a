"""TEST INFRASTRUCTURE: levels on the C oracle (oracle/), which has no level of its own.

A level s means that an episode plays world seed s: the reference's World.reset(seed=s) + generate_world, every
later draw keyed by s.  The oracle generates a world only in co_reset, from world_seed(env seed, episode).  For
a fixed env seed that hash is a bijection of the episode number modulo 2**64 up to its final `% (2**31 - 1)`, so
for every s there is an episode number whose world seed is exactly s (`episode_for`).  A scratch oracle env
resets there and generates world s; the env that plays the level imports that fresh state with its own episode
counter and world seed s (OracleEnv.import_state, the round trip the other oracle tests already rely on).  Envs
on level -1 reset as before.  Fresh worlds are cached by (geometry, s): level-replay runs draw from a few hundred
seeds."""
import functools

import numpy as np

from oracle import oracle_env

_M64 = (1 << 64) - 1
_P1, _P2, _P5 = 11400714785074694791, 14029467366897019727, 2870177450012600261
_TAIL = 2 ^ (_P5 ^ 3527539)  # the tuple hash's length term (co_world_seed, cr_common.h world_seed_of)
SCRATCH_SEED = 0


def _rotl31(v):
  return ((v << 31) | (v >> 33)) & _M64


def _rotr31(v):
  return ((v >> 31) | (v << 33)) & _M64


def episode_for(world_seed, seed=SCRATCH_SEED):
  """An episode number e (a signed 64-bit value) with world_seed(seed, e) == world_seed, for world_seed in
  [0, 2**31 - 2]: the hash's accumulator is made to end at world_seed itself, and every step of the hash before it
  (add, rotate, multiply by an odd constant, mod 2**64) is undone."""
  acc1 = _rotl31((_P5 + (seed & _M64) * _P2) & _M64) * _P1 & _M64  # after the seed lane
  acc2 = (world_seed - _TAIL) & _M64                                  # before the length term
  lane = (_rotr31(acc2 * pow(_P1, -1, 1 << 64) & _M64) - acc1) & _M64
  e = lane * pow(_P2, -1, 1 << 64) & _M64
  return e - (1 << 64) if e >> 63 else e


@functools.lru_cache(maxsize=None)
def _scratch(geometry):
  return oracle_env.OracleEnv(seed=SCRATCH_SEED, **dict(geometry))


@functools.lru_cache(maxsize=4096)
def fresh_world(world_seed, geometry):
  """The canonical state (OracleEnv.export_state) of a fresh episode on world seed `world_seed`; `geometry` is a
  tuple of the OracleEnv keyword items (area, view, size, length)."""
  episode = episode_for(world_seed)
  assert oracle_env.world_seed(SCRATCH_SEED, episode) == world_seed, world_seed
  env = _scratch(geometry)
  env.set_episode(episode - 1)  # co_reset counts it up first
  env.reset()
  return env.export_state()


def _key(kwargs):
  return tuple(sorted((k, tuple(v) if hasattr(v, '__len__') else v) for k, v in kwargs.items()))


def start_level(ref, world_seed, episode, geometry):
  """Start episode `episode` of oracle env `ref` on world seed `world_seed` (what reset() does on a level)."""
  ref.import_state(fresh_world(int(world_seed), geometry), 0, int(episode), int(world_seed))


class LevelEnv:
  """An OracleEnv with a level: reset() plays world seed `level` when it is >= 0, else the reference's sequence.
  The episode counter advances either way."""

  def __init__(self, seed=0, **kwargs):
    self.env = oracle_env.OracleEnv(seed=seed, **kwargs)
    self.seed, self.level, self.episode, self.world_seed = seed, -1, 0, 0
    self._geometry = _key(kwargs)

  def __getattr__(self, name):
    return getattr(self.env, name)

  def set_level(self, level):
    self.level = int(level)

  def reset(self):
    self.episode += 1
    if self.level >= 0:
      self.world_seed = self.level
      start_level(self.env, self.level, self.episode, self._geometry)
      return self.env.render()
    self.world_seed = oracle_env.world_seed(self.seed, self.episode)
    return self.env.reset()


class LevelBatch:
  """An OracleBatch with levels: reset(ids) starts the envs on level -1 through the batch, the others on their
  level's world.  Env i has seed seed + i."""

  def __init__(self, num_envs, seed=0, **kwargs):
    self.batch = oracle_env.OracleBatch(num_envs, seed=seed, **kwargs)
    self.level = np.full(num_envs, -1, np.int64)
    self.episode = np.zeros(num_envs, np.int64)
    self.seed = seed
    self._geometry = _key({k: v for k, v in kwargs.items() if k in ('area', 'view', 'size', 'length')})

  def __getattr__(self, name):
    return getattr(self.batch, name)

  def set_levels(self, levels, ids=None):
    """levels[k] for env ids[k] (all envs when ids is None)."""
    ids = np.arange(len(self.level)) if ids is None else np.asarray(ids, np.int64).reshape(-1)
    self.level[ids] = np.asarray(levels, np.int64).reshape(-1)

  def reset(self, ids=None, render=False):
    ids = np.arange(len(self.level)) if ids is None else np.asarray(ids, np.int64).reshape(-1)
    self.episode[ids] += 1
    on_level = self.level[ids] >= 0
    default = ids[~on_level]
    if len(default):
      self.batch.reset(default, render=False)
    for i in ids[on_level]:
      start_level(self.batch.envs[i], self.level[i], self.episode[i], self._geometry)
    if render:
      self.batch.obs[ids] = self.batch.render(ids)
    return self.batch.obs
