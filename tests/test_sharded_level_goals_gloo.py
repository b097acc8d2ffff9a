"""ShardedEnv with level goals (CPU, gloo, world_size 2): every rank registers the same table and goals, its LOCAL
envs sample from the table or are pinned, and each rank plays and counts its own episodes.  The ranks' episodes
(rewards and dones, gathered) and statistics (summed) equal one batch's, exactly.  The env behind it is
tests/test_level_goals.py's SimtGoalsEnv (the product's kernels on the SIMT emulator)."""
import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests.test_sharded_gloo import _free_port

K, T, LENGTH, SEED = 6, 30, 25, 41
TABLE = (np.array([4242, 17, 4242, 2 ** 31 - 2], np.int64), np.array([1, 2, 1, 0], np.int64))  # entries 0 and 2: one seed
PINNED = np.array([0, 1, 0, 0, 1, 0], bool)
ENTRIES = np.array([0, 3, 0, 0, 2, 0], np.int32)
GOALS = ('collect_sapling', 0, 'collect_wood', ['collect_sapling', 'collect_wood'])


class TorchSimtGoals:
  """SimtGoalsEnv with auto-reset and torch tensors out; set_level_table registers statistics as well."""

  def __init__(self, **kwargs):
    from tests.test_level_goals import SimtGoalsEnv
    self._e = SimtGoalsEnv(**kwargs)

  def reset(self, mask=None):
    return torch.from_numpy(self._e.reset(mask).copy())

  def set_level_table(self, seeds, weights=None):
    self._e.set_level_table(seeds, weights)
    self._e.set_level_stats()

  def set_level_goals(self, goals):
    from crafter_b200.env import goal_mask
    self._e.set_level_goals([goal_mask(g) for g in goals])

  def level_stats(self):
    return torch.from_numpy(self._e.stats.copy())

  def sample_levels(self, mask=None):
    self._e.sample_levels(mask)

  def pin_levels(self, entries, mask=None):
    self._e.pin_levels(entries, mask)

  def step(self, actions):
    obs, reward, done = self._e.step(np.asarray(actions))
    return torch.from_numpy(obs.copy()), torch.from_numpy(reward.copy()), torch.from_numpy(done.copy()), {}


def _play(env, mine):
  actions = np.random.RandomState(9).choice([1, 2, 3, 4, 5, 5, 5, 5], (T, K))
  env.set_level_table(*TABLE)
  env.set_level_goals(GOALS)
  env.sample_levels(~PINNED[mine])
  env.pin_levels(ENTRIES[mine], PINNED[mine])
  env.reset()
  rewards, dones = [], []
  for t in range(T):
    _, reward, done, _ = env.step(actions[t, mine])
    rewards.append(reward)
    dones.append(done)
  return env.level_stats(), torch.stack(rewards), torch.stack(dones)


def _worker(rank, world, port, shared):
  import os
  os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                    LOCAL_RANK=str(rank))
  dist.init_process_group('gloo', rank=rank, world_size=world)
  from crafter_b200.sharded import ShardedEnv
  env = ShardedEnv(num_envs=K, seed=SEED, env_factory=TorchSimtGoals, auto_reset=True, length=LENGTH)
  stats, rewards, dones = _play(env, env.local_slice())  # set_level_goals passes through to each shard
  dist.all_reduce(stats)
  parts = [torch.zeros_like(rewards) for _ in range(world)], [torch.zeros_like(dones, dtype=torch.uint8) for _ in range(world)]
  dist.all_gather(parts[0], rewards)
  dist.all_gather(parts[1], dones.to(torch.uint8))
  if rank == 0:
    shared['stats'] = stats.numpy()
    shared['rewards'] = torch.cat(parts[0], 1).numpy()
    shared['dones'] = torch.cat(parts[1], 1).numpy().astype(bool)
  dist.destroy_process_group()


def test_two_rank_goal_episodes_equal_one_batch():
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
  ref = TorchSimtGoals(num_envs=K, seed=SEED, auto_reset=True, length=LENGTH)
  want, rewards, dones = _play(ref, slice(0, K))
  assert (want.numpy() == got['stats']).all()
  assert (rewards.numpy() == got['rewards']).all() and (dones.numpy() == got['dones']).all()
  goal_rows = [0, 2, 3]
  assert (want[goal_rows, 3] % 10 == 0).all() and int(want[goal_rows, 3].sum()) > 0  # successes pay 1.0 each
