"""ShardedEnv with the level cache (CPU, gloo, world_size 2): every rank registers the same table and fills its own
cache of it; the shards gathered play what one batch without a cache plays, bit for bit.  The env behind it is
tests/test_level_cache.py's SimtCacheEnv (the product's kernels on the SIMT emulator)."""
import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests.test_sharded_gloo import _free_port
from tests.test_sharded_level_sampler_gloo import K, LATER, LENGTH, SAMPLED, SEED, TABLE, T

NEW_SEEDS = (10, np.array([4242, 17, 2 ** 31 - 2, 777, 99], np.int64))  # set_level_table with seed 0 replaced


class TorchSimtCache:
  """SimtCacheEnv with auto-reset and torch tensors out; set_level_cache / set_level_table behave as Env's."""

  def __init__(self, **kwargs):
    from tests.test_level_cache import SimtCacheEnv
    self._e = SimtCacheEnv(**kwargs)
    self._cached = False

  def reset(self, mask=None):
    return torch.from_numpy(self._e.reset(mask).copy())

  def set_level_table(self, seeds, weights=None):
    self._e.set_level_table(seeds, weights)
    if self._cached:  # the new buffers get their rows, filled where the seed changed
      self.set_level_cache()

  def set_level_cache(self, enabled=True):
    self._e.set_level_cache()
    self._e.fill()
    self._cached = True

  def set_level_weights(self, weights):
    self._e.set_level_weights(weights)

  def sample_levels(self, mask=None):
    self._e.sample_levels(mask)

  def step(self, actions):
    obs, reward, done = self._e.step(np.asarray(actions))
    info = {'final_observation': torch.from_numpy(self._e.final_obs.copy()),
            'final_world_seed': torch.from_numpy(self._e.final_world_seed.copy()),
            'world_seed': torch.from_numpy(self._e.world_seed())}
    return torch.from_numpy(obs.copy()), torch.from_numpy(reward.copy()), torch.from_numpy(done.copy()), info


def _play(env, mine, gather, cache):
  actions = np.random.RandomState(5).randint(0, 17, (T, K))
  env.set_level_table(*TABLE)
  if cache:
    env.set_level_cache()
  env.sample_levels(SAMPLED[mine])
  out = dict(obs=[gather(env.reset())], final=[], fws=[], ws=[], done=[])
  for t in range(T):
    if t == LATER[0]:
      env.set_level_weights(LATER[1])
      env.sample_levels(LATER[2][mine])
    if t == NEW_SEEDS[0]:
      env.set_level_table(NEW_SEEDS[1], LATER[1])
      env.sample_levels((SAMPLED | LATER[2])[mine])  # the new seed from the next episodes on
    obs, reward, done, info = env.step(actions[t, mine])
    full = gather(obs, info['final_observation'], info['final_world_seed'], info['world_seed'], done)
    for k, v in zip(('obs', 'final', 'fws', 'ws', 'done'), full):
      out[k].append(v)
  return {k: np.stack([x.numpy() for x in v]) for k, v in out.items()}


def _worker(rank, world, port, shared):
  import os
  os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                    LOCAL_RANK=str(rank))
  dist.init_process_group('gloo', rank=rank, world_size=world)
  from crafter_b200.sharded import ShardedEnv
  env = ShardedEnv(num_envs=K, seed=SEED, env_factory=TorchSimtCache, auto_reset=True, length=LENGTH)
  out = _play(env, env.local_slice(), env.gather, cache=True)  # set_level_cache passes through to each shard
  if rank == 0:
    shared.update(out)
  dist.destroy_process_group()


def test_two_rank_cached_shards_equal_one_uncached_batch():
  ctx = mp.get_context('spawn')  # never fork a multi-threaded pytest process
  manager = ctx.Manager()
  got = manager.dict()
  port = _free_port()
  procs = [ctx.Process(target=_worker, args=(r, 2, port, got)) for r in range(2)]
  for p in procs:
    p.start()
  for p in procs:
    p.join(300)
    assert p.exitcode == 0
  ref = TorchSimtCache(num_envs=K, seed=SEED, auto_reset=True, length=LENGTH)
  want = _play(ref, slice(0, K), lambda *tensors: tensors[0] if len(tensors) == 1 else tensors, cache=False)
  for k, v in want.items():
    assert (v == got[k]).all(), k
  assert want['done'].sum() >= 2 * K, 'the run should cross several auto-resets'
  assert 777 in set(want["ws"].ravel().tolist()), "the replaced seed was never played"
