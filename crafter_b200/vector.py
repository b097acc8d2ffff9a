"""Gymnasium vector-env adaptor over `crafter_b200.Env` and the reference's gym ids
(crafter/__init__.py:4-17: `CrafterReward-v1`, `CrafterNoReward-v1`, max 10000 steps).

    venv = crafter_b200.vector.make('CrafterReward-v1', num_envs=4096, seed=0)
    obs, info = venv.reset()
    obs, reward, terminated, truncated, info = venv.step(actions)     # torch.cuda tensors

It follows `gymnasium.vector.VectorEnv` (1.x): batched `observation_space` / `action_space` next to
`single_*`, `reset(seed=, options=)`, the five-tuple `step`, `metadata['autoreset_mode']`.  The batch
resets inside the step that ends an episode (gymnasium's SAME_STEP mode: `obs` is the first frame of
the next episode), and the terminal transition travels in `info` under gymnasium's keys:

    info['final_obs'][i], info['final_info'][...][i]   valid where info['_final_obs'][i] (= done)

(`final_observation` / `_final_observation` are kept as aliases for gymnasium <= 0.29 code.)
`terminated` = the player died (`discount` 0 in the reference, env.py:105,111) or reached its level goal
(Env.set_level_goals: `discount` 0 too, success ends the task), `truncated` = the episode hit `length` (the
registration's max_episode_steps).  `reset(options={'levels': levels})` (with or
without 'reset_mask') and `set_levels(levels, mask)` choose the worlds the episodes play (Env.set_levels);
`set_level_table`, `set_level_weights` and `sample_levels` make envs draw them from a weighted table inside the step
(Env.set_level_table).  Arrays are torch.cuda tensors unless
`to_numpy=True`.  With `observation='semantic'` (see `crafter_b200.Env`) the observations, `final_obs`
included, are the local semantic windows and the spaces say so (`Box(0, 18, (gx, gy), uint8)`); with
`observation='symbolic'` they are the symbolic vectors (`Box(0, 1, (D,), float32)`).
gym / gymnasium are optional (absent in this image): with gymnasium installed the
class derives from `gymnasium.vector.VectorEnv` and uses its spaces; `register()` adds the two ids
when either package is importable.
"""
import numpy as np

IDS = {'CrafterReward-v1': dict(reward=True), 'CrafterNoReward-v1': dict(reward=False)}

try:  # optional
  import gymnasium as _gym
  _Base = _gym.vector.VectorEnv
except Exception:  # noqa: BLE001 (any import problem of an optional package)
  _gym, _Base = None, object


class _Box:
  """Stand-in for gymnasium.spaces.Box when gymnasium is not installed."""

  def __init__(self, low, high, shape, dtype):
    self.low, self.high, self.shape, self.dtype = low, high, tuple(shape), np.dtype(dtype)

  def sample(self):
    if self.dtype.kind == 'f':
      return np.random.uniform(self.low, self.high, self.shape).astype(self.dtype)
    return np.random.randint(self.low, self.high + 1, self.shape).astype(self.dtype)

  def contains(self, x):
    x = np.asarray(x)
    return x.shape == self.shape and bool((x >= self.low).all() and (x <= self.high).all())

  def __repr__(self):
    return f'Box({self.low}, {self.high}, {self.shape}, {self.dtype})'


class _Discrete:

  def __init__(self, n):
    self.n, self.shape, self.dtype = int(n), (), np.dtype(np.int64)

  def sample(self):
    return int(np.random.randint(self.n))

  def contains(self, x):
    return 0 <= int(x) < self.n

  def __repr__(self):
    return f'Discrete({self.n})'


class _MultiDiscrete:

  def __init__(self, nvec):
    self.nvec = np.asarray(nvec, np.int64)
    self.shape, self.dtype = self.nvec.shape, np.dtype(np.int64)

  def sample(self):
    return (np.random.random(self.shape) * self.nvec).astype(np.int64)

  def contains(self, x):
    x = np.asarray(x)
    return x.shape == self.shape and bool((x >= 0).all() and (x < self.nvec).all())

  def __repr__(self):
    return f'MultiDiscrete({self.nvec.tolist()[:4]}...)'


def _spaces(num_envs, obs_shape, n_actions, high=255, dtype=np.uint8):
  if _gym is not None:
    sp = _gym.spaces
    single_obs = sp.Box(0, high, obs_shape, dtype)
    single_act = sp.Discrete(n_actions)
    return (single_obs, single_act, _gym.vector.utils.batch_space(single_obs, num_envs),
            _gym.vector.utils.batch_space(single_act, num_envs))
  return (_Box(0, high, obs_shape, dtype), _Discrete(n_actions),
          _Box(0, high, (num_envs,) + tuple(obs_shape), dtype), _MultiDiscrete([n_actions] * num_envs))


class VectorEnv(_Base):
  """`gymnasium.vector.VectorEnv` over one batched `crafter_b200.Env` (no sub-environments: the batch
  IS the environment)."""

  def __init__(self, num_envs, to_numpy=False, final_obs=True, **kwargs):
    from .env import Env
    kwargs.setdefault('auto_reset', True)
    if not kwargs['auto_reset']:
      final_obs = False
    self.env = Env(num_envs=num_envs, final_obs=final_obs, **kwargs)
    self.num_envs = self.env.num_envs
    self._to_numpy = bool(to_numpy)
    self._final = bool(final_obs)
    (self.single_observation_space, self.single_action_space, self.observation_space,
     self.action_space) = _spaces(self.num_envs, self.env.observation_space.shape, self.env.action_space.n,
                                  self.env.observation_space.high, self.env.observation_space.dtype)
    mode = 'same_step' if kwargs['auto_reset'] else 'disabled'
    if _gym is not None and hasattr(_gym.vector, 'AutoresetMode'):
      mode = _gym.vector.AutoresetMode(mode)
    self.metadata = {'render_modes': ['rgb_array'], 'autoreset_mode': mode}
    self.render_mode = 'rgb_array'
    self.spec = None
    self.closed = False

  def _out(self, x):
    return x.cpu().numpy() if self._to_numpy else x

  def reset(self, *, seed=None, options=None):
    if seed is not None and int(seed) != self.env._seed:
      raise ValueError('the seed is fixed at construction (per-episode seeds derive from it and the env index); '
                       'make a new VectorEnv to change it')
    options = options or {}
    mask = options.get('reset_mask')  # gymnasium 1.x: partial resets through options
    # the world seeds of the episodes this reset starts (Env.set_levels; -1 = the reference's sequence)
    return self._out(self.env.reset(mask, options.get('levels'))), {}

  def set_levels(self, levels, mask=None):
    """Env.set_levels: the worlds of the envs' next episodes."""
    self.env.set_levels(levels, mask)

  def set_level_table(self, seeds, weights=None):
    """Env.set_level_table: the weighted table of world seeds the sampled envs draw from."""
    self.env.set_level_table(seeds, weights)

  def set_level_weights(self, weights):
    """Env.set_level_weights: new weights for the table's seeds (no host read with a device tensor)."""
    self.env.set_level_weights(weights)

  def sample_levels(self, mask=None):
    """Env.sample_levels: these envs draw the world of every new episode from the level table."""
    self.env.sample_levels(mask)

  def set_level_cache(self, enabled=True):
    """Env.set_level_cache: keep the level table's worlds generated on the device (memory for time)."""
    self.env.set_level_cache(enabled)

  def author_levels(self, entries, materials, creatures=None):
    """Env.author_levels: caller-made worlds into level table entries."""
    self.env.author_levels(entries, materials, creatures)

  def level_worlds(self, entries):
    """Env.level_worlds: the worlds the level cache holds for these entries."""
    return self.env.level_worlds(entries)

  def mutate_levels(self, parents, children, edits, key, weights=None):
    """Env.mutate_levels: children of level table entries, made by keyed random edits of their worlds."""
    return self.env.mutate_levels(parents, children, edits, key, weights)

  def pin_levels(self, entries, mask=None):
    """Env.pin_levels: these envs play one level table entry in every new episode."""
    self.env.pin_levels(entries, mask)

  def set_level_stats(self, enabled=True):
    """Env.set_level_stats: count every finished episode against the level table entry it was drawn from."""
    self.env.set_level_stats(enabled)

  def level_stats(self):
    """Env.level_stats: copies of the per-entry episode statistics."""
    return self.env.level_stats()

  def clear_level_stats(self, entries=None):
    """Env.clear_level_stats: zero the statistics of these entries (None: all)."""
    self.env.clear_level_stats(entries)

  def set_level_goals(self, goals):
    """Env.set_level_goals: achievement goals per level table entry that pay the reward and end the episode."""
    self.env.set_level_goals(goals)

  @property
  def level_goals(self):
    """Env.level_goals: a copy of the goal masks of the table entries in use, or None."""
    return self.env.level_goals

  def set_level_starts(self, starts):
    """Env.set_level_starts: the player's start position, facing, inventory and vitals per level table entry."""
    self.env.set_level_starts(starts)

  @property
  def level_starts(self):
    """Env.level_starts: a copy of the start records of the table entries in use, or None."""
    return self.env.level_starts

  def step(self, actions):
    obs, reward, done, info = self.env.step(actions)
    dead = self.env.state['final_stats'][:, 23] != 0
    terminated, truncated = done & dead, done & ~dead
    out = {'reward': info['reward'], 'discount': info['discount'], 'inventory': info['inventory'],
           'achievements': info['achievements'], 'player_pos': info['player_pos']}
    if self.env._auto_reset:  # the terminal transition of the envs that were regenerated inside the step
      final_info = {'inventory': info['final_inventory'], 'achievements': info['final_achievements'],
                    'player_pos': info['final_player_pos'],
                    'discount': info['discount'], 'reward': info['reward']}
      out['final_info'], out['_final_info'] = final_info, done
      if self._final:
        out['final_obs'] = out['final_observation'] = info['final_observation']
        out['_final_obs'] = out['_final_observation'] = done
    if self._to_numpy:
      conv = lambda v: {k: conv(x) for k, x in v.items()} if isinstance(v, dict) else v.cpu().numpy()
      out = {k: conv(v) for k, v in out.items()}
    return self._out(obs), self._out(reward), self._out(terminated), self._out(truncated), out

  def render(self):
    return self._out(self.env.render())

  def close(self, **kwargs):
    if not self.closed:
      self.env.close()
      self.closed = True

  @property
  def unwrapped(self):
    return self


def make(env_id, num_envs, **kwargs):
  spec = dict(IDS[env_id])
  spec.setdefault('length', 10000)  # max_episode_steps of the reference registration
  spec.update(kwargs)
  return VectorEnv(num_envs, **spec)


def register():
  """Register the reference's ids (crafter/__init__.py:6-15) with gymnasium / gym when installed: as vector
  entry points (`gymnasium.make_vec(id, num_envs=...)`) and, for `gymnasium.make(id)`, as a batch of one."""
  done = []
  for modname in ('gymnasium', 'gym'):
    try:
      mod = __import__(modname)
    except ImportError:
      continue
    for env_id, spec in IDS.items():
      vec = lambda num_envs=1, _id=env_id, **kw: make(_id, num_envs, **kw)
      try:
        mod.register(id=env_id, entry_point=lambda _id=env_id, **kw: make(_id, 1, **kw),
                     vector_entry_point=vec, max_episode_steps=10000)
        done.append((modname, env_id))
      except TypeError:  # an older API without vector entry points
        try:
          mod.register(id=env_id, entry_point=lambda _id=env_id, **kw: make(_id, 1, **kw), max_episode_steps=10000)
          done.append((modname, env_id))
        except Exception:  # noqa: BLE001
          pass
      except Exception:  # noqa: BLE001 (already registered)
        pass
  return done
