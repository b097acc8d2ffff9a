"""ShardedEnv with the level sampler (CPU, gloo, world_size 2): every rank registers the same table, the mask of
sample_levels is the local shard's, and since the draw is keyed by the global env index the shards' frames,
terminal frames and world seeds gathered equal one big batch bit for bit.  The env behind it is
tests/test_level_sampler.py's SimtSamplerEnv (the product's kernels on the SIMT emulator)."""
import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests.test_sharded_gloo import _free_port

K, T, LENGTH, SEED = 6, 24, 5, 13
TABLE = (np.array([4242, 17, 2 ** 31 - 2, 0, 99], np.int64), np.array([2, 1, 1, 0, 3], np.int64))
SAMPLED = np.array([1, 0, 1, 1, 0, 1], bool)  # at reset; the others play the reference's sequence
LATER = (9, np.array([0, 0, 0, 5, 1], np.int64), np.array([0, 1, 0, 0, 1, 0], bool))  # new weights, more sampled envs


class TorchSimtSampler:
  """SimtSamplerEnv with auto-reset and torch tensors out (what ShardedEnv.gather expects)."""

  def __init__(self, **kwargs):
    from tests.test_level_sampler import SimtSamplerEnv
    self._e = SimtSamplerEnv(**kwargs)

  def reset(self, mask=None):
    return torch.from_numpy(self._e.reset(mask).copy())

  def set_level_table(self, seeds, weights=None):
    self._e.set_level_table(seeds, weights)

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


def _play(env, mine, gather):
  actions = np.random.RandomState(5).randint(0, 17, (T, K))
  env.set_level_table(*TABLE)
  env.sample_levels(SAMPLED[mine])
  out = dict(obs=[gather(env.reset())], final=[], fws=[], ws=[], done=[])
  for t in range(T):
    if t == LATER[0]:
      env.set_level_weights(LATER[1])
      env.sample_levels(LATER[2][mine])
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
  env = ShardedEnv(num_envs=K, seed=SEED, env_factory=TorchSimtSampler, auto_reset=True, length=LENGTH)
  out = _play(env, env.local_slice(), env.gather)
  if rank == 0:
    shared.update(out)
  dist.destroy_process_group()


def test_two_rank_sampler_shards_equal_one_batch():
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
  ref = TorchSimtSampler(num_envs=K, seed=SEED, auto_reset=True, length=LENGTH)
  want = _play(ref, slice(0, K), lambda *tensors: tensors[0] if len(tensors) == 1 else tensors)
  for k, v in want.items():
    assert (v == got[k]).all(), k
  assert want['done'].sum() >= 2 * K, 'the run should cross several auto-resets'
  played = set(want['fws'][want['done']].tolist())
  assert len(played & set(TABLE[0].tolist())) >= 3, played
  late = want['ws'][-1][SAMPLED | LATER[2]]
  assert set(late.tolist()) <= {0, 99}, late  # only the seeds of the later weights are left by the end of the run
