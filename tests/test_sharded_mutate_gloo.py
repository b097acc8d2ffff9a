"""ShardedEnv with level mutation (CPU, gloo, world_size 2): every rank registers the same table and makes the same
mutate_levels call into its own cache, with nothing broadcast.  The ranks' rows come out identical, and the shards
gathered then play what one batch plays, bit for bit.  The env behind it is tests/test_mutate_levels.py's
SimtMutateEnv (the product's kernels on the SIMT emulator)."""
import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests.test_sharded_gloo import _free_port

K, T, LENGTH, SEED = 6, 16, 4, 31
TABLE = np.array([4242, 17, 2 ** 31 - 2, 4242, 17], np.int64)
PARENTS, CHILDREN, EDITS, KEY = [0, 1, 3], [3, 4, 0], 300, 0xABCDEF
WEIGHTS = {'cow': 2, 'zombie': 2, 'skeleton': 1, 'stone': 1, 'tree': 1, 'path': 1, 'remove': 1}
ENTRIES = np.array([3, 4, 0, 2, 3, 4], np.int32)


class TorchSimtMutate:
  """SimtMutateEnv with auto-reset and torch tensors out; mutate_levels / pin_levels behave as Env's."""

  def __init__(self, **kwargs):
    from tests.test_mutate_levels import SimtMutateEnv
    self._e = SimtMutateEnv(**kwargs)

  def reset(self, mask=None):
    return torch.from_numpy(self._e.reset(mask).copy())

  def set_level_table(self, seeds, weights=None):
    self._e.set_level_table(seeds, weights)
    self._e.set_level_cache()
    self._e.fill()

  def mutate_levels(self, parents, children, edits, key, weights=None):
    worlds, status = self._e.mutate(parents, children, edits, key, weights)
    assert (status == 0).all(), status
    W, H = self._e.area
    w = torch.from_numpy(worlds).reshape(-1, W, H)
    return dict(materials=w & 15, creatures=w >> 4)

  def rows(self):
    return self._e.rows()

  def pin_levels(self, entries, mask=None):
    self._e.pin_levels(entries, mask)

  def step(self, actions):
    obs, reward, done = self._e.step(np.asarray(actions))
    info = {'final_observation': torch.from_numpy(self._e.final_obs.copy()),
            'final_world_seed': torch.from_numpy(self._e.final_world_seed.copy())}
    return torch.from_numpy(obs.copy()), torch.from_numpy(reward.copy()), torch.from_numpy(done.copy()), info


def _play(env, mine, gather):
  actions = np.random.RandomState(5).randint(0, 17, (T, K))
  env.set_level_table(TABLE)
  children = env.mutate_levels(PARENTS, CHILDREN, EDITS, KEY, WEIGHTS)  # the same call on every rank
  rows = env.rows()
  env.pin_levels(ENTRIES[mine])
  out = dict(obs=[gather(env.reset())], final=[], fws=[], done=[])
  for t in range(T):
    obs, reward, done, info = env.step(actions[t, mine])
    full = gather(obs, info['final_observation'], info['final_world_seed'], done)
    for k, v in zip(('obs', 'final', 'fws', 'done'), full):
      out[k].append(v)
  played = {k: np.stack([x.numpy() for x in v]) for k, v in out.items()}
  return played, rows, {k: v.numpy() for k, v in children.items()}


def _worker(rank, world, port, shared):
  import os
  os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                    LOCAL_RANK=str(rank))
  dist.init_process_group('gloo', rank=rank, world_size=world)
  from crafter_b200.sharded import ShardedEnv
  env = ShardedEnv(num_envs=K, seed=SEED, env_factory=TorchSimtMutate, auto_reset=True, length=LENGTH)
  played, rows, children = _play(env, env.local_slice(), env.gather)  # mutate_levels passes through to each shard
  shared[f'rows{rank}'] = rows
  shared[f'children{rank}'] = children
  if rank == 0:
    shared['played'] = played
  dist.destroy_process_group()


def test_two_ranks_make_the_same_children_and_play_one_batch():
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
  assert all((a == b).all() for a, b in zip(got['rows0'], got['rows1'])), 'the ranks made different rows'
  for k in ('materials', 'creatures'):
    assert (got['children0'][k] == got['children1'][k]).all(), k
  ref = TorchSimtMutate(num_envs=K, seed=SEED, auto_reset=True, length=LENGTH)
  want, rows, _ = _play(ref, slice(0, K), lambda *tensors: tensors[0] if len(tensors) == 1 else tensors)
  assert all((a == b).all() for a, b in zip(rows, got['rows0']))
  for k, v in want.items():
    assert (v == got['played'][k]).all(), k
  assert want['done'].sum() >= 2 * K, 'the run should cross several auto-resets'
  assert set(want['fws'][want['done'].astype(bool)].tolist()) <= set(TABLE.tolist())
