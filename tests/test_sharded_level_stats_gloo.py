"""ShardedEnv with per-level episode statistics (CPU, gloo, world_size 2): every rank registers the same table, its
LOCAL envs sample from it or are pinned, and each rank counts its own episodes.  The ranks' statistics summed (an
all-reduce) equal what one batch counts, exactly.  The env behind it is tests/test_level_stats.py's SimtStatsEnv
(the product's kernels on the SIMT emulator)."""
import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests.test_sharded_gloo import _free_port

K, T, LENGTH, SEED = 6, 18, 3, 41
TABLE = (np.array([4242, 17, 4242, 2 ** 31 - 2], np.int64), np.array([1, 2, 1, 0], np.int64))  # entries 0 and 2: one seed
PINNED = np.array([0, 1, 0, 0, 1, 0], bool)
ENTRIES = np.array([0, 3, 0, 0, 2, 0], np.int32)


class TorchSimtStats:
  """SimtStatsEnv with auto-reset and torch tensors out; set_level_table registers the notes as Env's does."""

  def __init__(self, **kwargs):
    from tests.test_level_stats import SimtStatsEnv
    self._e = SimtStatsEnv(**kwargs)

  def reset(self, mask=None):
    return torch.from_numpy(self._e.reset(mask).copy())

  def set_level_table(self, seeds, weights=None):
    self._e.set_level_table(seeds, weights)
    self._e.set_level_stats()

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
  actions = np.random.RandomState(9).randint(0, 17, (T, K))
  env.set_level_table(*TABLE)
  env.sample_levels(~PINNED[mine])
  env.pin_levels(ENTRIES[mine], PINNED[mine])
  env.reset()
  done = 0
  for t in range(T):
    done += int(env.step(actions[t, mine])[2].sum())
  return env.level_stats(), done


def _worker(rank, world, port, shared):
  import os
  os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                    LOCAL_RANK=str(rank))
  dist.init_process_group('gloo', rank=rank, world_size=world)
  from crafter_b200.sharded import ShardedEnv
  env = ShardedEnv(num_envs=K, seed=SEED, env_factory=TorchSimtStats, auto_reset=True, length=LENGTH)
  stats, _ = _play(env, env.local_slice())  # level_stats passes through to each shard
  dist.all_reduce(stats)
  if rank == 0:
    shared['stats'] = stats.numpy()
  dist.destroy_process_group()


def test_two_rank_stats_sum_to_one_batch():
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
  ref = TorchSimtStats(num_envs=K, seed=SEED, auto_reset=True, length=LENGTH)
  want, done = _play(ref, slice(0, K))
  assert (want.numpy() == got['stats']).all()
  assert done >= 2 * K and int(want[:, 0].sum()) == done
  assert want[0, 0] > 0 and want[2, 0] > 0 and want[3, 0] > 0  # one seed, two entries; a weight-0 pinned entry
