"""ShardedEnv with authored levels and pinning (CPU, gloo, world_size 2): every rank registers the same table and
authors the same worlds into its own cache; each rank pins and samples its LOCAL envs.  The shards gathered play
what one batch plays, bit for bit.  The env behind it is tests/test_authored_levels.py's SimtAuthoredEnv (the
product's kernels on the SIMT emulator)."""
import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests.test_sharded_gloo import _free_port

K, T, LENGTH, SEED = 6, 16, 4, 29
TABLE = (np.array([4242, 17, 2 ** 31 - 2], np.int64), np.array([1, 0, 2], np.int64))
PINNED = np.array([1, 0, 1, 0, 1, 1], bool)
ENTRIES = np.array([1, 0, 0, 0, 2, 1], np.int32)  # entry 1 has weight 0: only pinned envs play it


def worlds():
  """Two authored worlds (entries 0 and 1): lava, sand and path around the start, a few creatures."""
  from tests.test_authored_levels import COW, GRASS, LAVA, PATH, SAND, ZOMBIE
  m = np.full((2, 64, 64), GRASS, np.int64)
  c = np.zeros((2, 64, 64), np.int64)
  m[0, 31, 32], m[0, 40:, :] = LAVA, SAND
  c[0, 33, 32], c[0, 50, 9] = ZOMBIE, COW
  m[1, :, 30:34] = PATH
  c[1, 20, 31] = COW
  return m, c


class TorchSimtAuthored:
  """SimtAuthoredEnv with auto-reset and torch tensors out; author_levels / pin_levels behave as Env's."""

  def __init__(self, **kwargs):
    from tests.test_authored_levels import SimtAuthoredEnv
    self._e = SimtAuthoredEnv(**kwargs)

  def reset(self, mask=None):
    return torch.from_numpy(self._e.reset(mask).copy())

  def set_level_table(self, seeds, weights=None):
    self._e.set_level_table(seeds, weights)

  def author_levels(self, entries, materials, creatures=None):
    from tests.test_authored_levels import pack
    self._e.set_level_cache()
    self._e.fill()
    assert (self._e.author(entries, pack(materials, creatures)) == 0).all()

  def sample_levels(self, mask=None):
    self._e.sample_levels(mask)

  def pin_levels(self, entries, mask=None):
    self._e.pin_levels(entries, mask)

  def step(self, actions):
    obs, reward, done = self._e.step(np.asarray(actions))
    info = {'final_observation': torch.from_numpy(self._e.final_obs.copy()),
            'final_world_seed': torch.from_numpy(self._e.final_world_seed.copy()),
            'world_seed': torch.from_numpy(self._e.world_seed())}
    return torch.from_numpy(obs.copy()), torch.from_numpy(reward.copy()), torch.from_numpy(done.copy()), info


def _play(env, mine, gather):
  actions = np.random.RandomState(5).randint(0, 17, (T, K))
  env.set_level_table(*TABLE)
  env.author_levels([0, 1], *worlds())  # the same worlds on every rank, like the table
  env.sample_levels(~PINNED[mine])
  env.pin_levels(ENTRIES[mine], PINNED[mine])
  out = dict(obs=[gather(env.reset())], final=[], fws=[], ws=[], done=[])
  for t in range(T):
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
  env = ShardedEnv(num_envs=K, seed=SEED, env_factory=TorchSimtAuthored, auto_reset=True, length=LENGTH)
  out = _play(env, env.local_slice(), env.gather)  # author_levels and pin_levels pass through to each shard
  if rank == 0:
    shared.update(out)
  dist.destroy_process_group()


def test_two_rank_authored_shards_equal_one_batch():
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
  ref = TorchSimtAuthored(num_envs=K, seed=SEED, auto_reset=True, length=LENGTH)
  want = _play(ref, slice(0, K), lambda *tensors: tensors[0] if len(tensors) == 1 else tensors)
  for k, v in want.items():
    assert (v == got[k]).all(), k
  assert want['done'].sum() >= 2 * K, 'the run should cross several auto-resets'
  ws = want['ws']
  assert set(ws[:, PINNED].ravel().tolist()) == set(TABLE[0].tolist()) and 17 not in set(ws[:, ~PINNED].ravel().tolist())
