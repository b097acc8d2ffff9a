"""ShardedEnv with levels (CPU, gloo, world_size 2): levels are local to the shard, like actions, and the shards'
frames, terminal frames and final world seeds gathered equal one big batch with the same levels bit for bit.
The env behind it is tests/test_levels.py's SimtLevelsEnv (the product's kernels on the SIMT emulator)."""
import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests.test_sharded_gloo import _free_port

K, T, LENGTH, SEED = 6, 24, 5, 13
LEVELS = np.array([-1, 4242, 0, 4242, -1, 2 ** 31 - 2], np.int32)  # at reset
LATER = (9, np.array([77, -1, -1, 5, 4242, -1], np.int32), np.array([1, 1, 0, 1, 1, 0], bool))  # set_levels at step 9


class TorchSimtLevels:
  """SimtLevelsEnv with auto-reset and torch tensors out (what ShardedEnv.gather expects)."""

  def __init__(self, **kwargs):
    from tests.test_levels import SimtLevelsEnv
    self._e = SimtLevelsEnv(**kwargs)

  def reset(self, mask=None, levels=None):
    return torch.from_numpy(self._e.reset(mask, levels).copy())

  def set_levels(self, levels, mask=None):
    self._e.set_levels(levels, mask)

  def step(self, actions):
    obs, reward, done = self._e.step(np.asarray(actions))
    info = {'final_observation': torch.from_numpy(self._e.final_obs.copy()),
            'final_world_seed': torch.from_numpy(self._e.final_world_seed.copy()),
            'world_seed': torch.from_numpy(self._e.world_seed())}
    return torch.from_numpy(obs.copy()), torch.from_numpy(reward.copy()), torch.from_numpy(done.copy()), info


def _worker(rank, world, port, shared):
  import os
  os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                    LOCAL_RANK=str(rank))
  dist.init_process_group('gloo', rank=rank, world_size=world)
  from crafter_b200.sharded import ShardedEnv
  env = ShardedEnv(num_envs=K, seed=SEED, env_factory=TorchSimtLevels, auto_reset=True, length=LENGTH)
  mine = env.local_slice()
  actions = np.random.RandomState(5).randint(0, 17, (T, K))
  out = dict(obs=[env.gather(env.reset(levels=LEVELS[mine]))], final=[], fws=[], ws=[])
  for t in range(T):
    if t == LATER[0]:
      env.set_levels(LATER[1][mine], LATER[2][mine])
    obs, reward, done, info = env.step(actions[t, mine])
    full = env.gather(obs, info['final_observation'], info['final_world_seed'], info['world_seed'])
    for k, v in zip(('obs', 'final', 'fws', 'ws'), full):
      out[k].append(v)
  if rank == 0:
    for k, v in out.items():
      shared[k] = np.stack([x.numpy() for x in v])
  dist.destroy_process_group()


def test_two_rank_level_shards_equal_one_batch():
  from tests.test_levels import SimtLevelsEnv
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
  ref = SimtLevelsEnv(num_envs=K, seed=SEED, auto_reset=True, length=LENGTH)
  actions = np.random.RandomState(5).randint(0, 17, (T, K))
  want = dict(obs=[ref.reset(levels=LEVELS).copy()], final=[], fws=[], ws=[])
  dones = []
  for t in range(T):
    if t == LATER[0]:
      ref.set_levels(LATER[1], LATER[2])
    obs, _, done = ref.step(actions[t])
    want['obs'].append(obs.copy()); want['final'].append(ref.final_obs.copy())
    want['fws'].append(ref.final_world_seed.copy()); want['ws'].append(ref.world_seed())
    dones.append(done.copy())
  for k, v in want.items():
    assert (np.stack(v) == got[k]).all(), k
  assert np.stack(dones).sum() >= 2 * K, 'the run should cross several auto-resets'
  assert {4242, 77, 5} <= set(np.stack(want['fws']).ravel().tolist())
