"""ShardedEnv with level starts (CPU, gloo, world_size 2): every rank registers the same table and starts, its LOCAL
envs sample from the table or are pinned, and each rank plays its own episodes.  The ranks' episodes (rewards, dones
and the players' positions and inventories, gathered) equal one batch's, exactly.  The env behind it is
tests/test_level_starts.py's SimtStartsEnv (the product's kernels on the SIMT emulator)."""
import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests.test_sharded_gloo import _free_port

K, T, LENGTH, SEED = 6, 30, 9, 41
TABLE = (np.array([4242, 17, 4242, 2 ** 31 - 2], np.int64), np.array([1, 2, 1, 0], np.int64))  # entries 0 and 2: one seed
PINNED = np.array([0, 1, 0, 0, 1, 0], bool)
ENTRIES = np.array([0, 3, 0, 0, 2, 0], np.int32)
STARTS = (dict(inventory={'wood_pickaxe': 1, 'food': 2}, pos=(33, 31), facing='up'), None,
          dict(inventory={'health': 4}, pos=(30, 33), facing='left'), dict(pos=(34, 32), facing=(1, 0)))


class TorchSimtStarts:
  """SimtStartsEnv with auto-reset and torch tensors out."""

  def __init__(self, **kwargs):
    from tests.test_level_starts import SimtStartsEnv
    self._e = SimtStartsEnv(**kwargs)

  def reset(self, mask=None):
    return torch.from_numpy(self._e.reset(mask).copy())

  def set_level_table(self, seeds, weights=None):
    self._e.set_level_table(seeds, weights)

  def set_level_starts(self, starts):
    from crafter_b200.env import START_WORDS, level_start
    self._e.set_level_starts([np.zeros(START_WORDS, np.int32) if s is None else level_start(**s) for s in starts])

  def sample_levels(self, mask=None):
    self._e.sample_levels(mask)

  def pin_levels(self, entries, mask=None):
    self._e.pin_levels(entries, mask)

  def player(self):
    return torch.from_numpy(np.concatenate([self._e.state['inventory'], self._e.state['pstate'][:, 12:14]], 1))

  def step(self, actions):
    obs, reward, done = self._e.step(np.asarray(actions))
    return torch.from_numpy(obs.copy()), torch.from_numpy(reward.copy()), torch.from_numpy(done.copy()), {}


def _play(env, mine):
  actions = np.random.RandomState(9).randint(0, 17, (T, K))
  env.set_level_table(*TABLE)
  env.set_level_starts(STARTS)
  env.sample_levels(~PINNED[mine])
  env.pin_levels(ENTRIES[mine], PINNED[mine])
  env.reset()
  rewards, dones, players = [], [], [env.player()]
  for t in range(T):
    _, reward, done, _ = env.step(actions[t, mine])
    rewards.append(reward)
    dones.append(done)
    players.append(env.player())
  return torch.stack(rewards), torch.stack(dones), torch.stack(players)


def _worker(rank, world, port, shared):
  import os
  os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                    LOCAL_RANK=str(rank))
  dist.init_process_group('gloo', rank=rank, world_size=world)
  from crafter_b200.sharded import ShardedEnv
  env = ShardedEnv(num_envs=K, seed=SEED, env_factory=TorchSimtStarts, auto_reset=True, length=LENGTH)
  rewards, dones, players = _play(env, env.local_slice())  # set_level_starts passes through to each shard
  parts = ([torch.zeros_like(rewards) for _ in range(world)], [torch.zeros_like(dones, dtype=torch.uint8) for _ in range(world)],
           [torch.zeros_like(players) for _ in range(world)])
  dist.all_gather(parts[0], rewards)
  dist.all_gather(parts[1], dones.to(torch.uint8))
  dist.all_gather(parts[2], players)
  if rank == 0:
    shared['rewards'] = torch.cat(parts[0], 1).numpy()
    shared['dones'] = torch.cat(parts[1], 1).numpy().astype(bool)
    shared['players'] = torch.cat(parts[2], 1).numpy()
  dist.destroy_process_group()


def test_two_rank_start_episodes_equal_one_batch():
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
  ref = TorchSimtStarts(num_envs=K, seed=SEED, auto_reset=True, length=LENGTH)
  rewards, dones, players = _play(ref, slice(0, K))
  assert (rewards.numpy() == got['rewards']).all() and (dones.numpy() == got['dones']).all()
  assert (players.numpy() == got['players']).all()
  assert dones.any() and ((players[:, :, 16] != 32) | (players[:, :, 17] != 32)).any()  # episodes started off-centre
