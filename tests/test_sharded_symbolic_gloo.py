"""ShardedEnv over symbolic vectors (CPU, gloo, world_size 2): `gather` reassembles float32 vectors, terminal
vectors included, into the vectors of the single-process batch bit for bit.  The env behind it is
observation='symbolic' on the SIMT emulator (tests/test_symbolic_obs.py)."""
import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests.test_sharded_gloo import _free_port

K, T, LENGTH = 4, 30, 20


class TorchSimtSymbolic:
  """SimtSymbolicEnv with torch tensors out (what ShardedEnv.gather expects)."""

  def __init__(self, **kwargs):
    from tests.test_symbolic_obs import SimtSymbolicEnv
    self._e = SimtSymbolicEnv(final_obs=True, **kwargs)

  def reset(self, mask=None):
    return torch.from_numpy(self._e.reset(mask).copy())

  def step(self, actions):
    vec, reward, done = self._e.step(np.asarray(actions))
    info = {'final_observation': torch.from_numpy(self._e.final_symbolic.copy())}
    return torch.from_numpy(vec.copy()), torch.from_numpy(reward.copy()), torch.from_numpy(done.copy()), info


def _worker(rank, world, port, shared):
  import os
  os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                    LOCAL_RANK=str(rank))
  dist.init_process_group('gloo', rank=rank, world_size=world)
  from crafter_b200.sharded import ShardedEnv
  env = ShardedEnv(num_envs=K, seed=11, env_factory=TorchSimtSymbolic, auto_reset=True, length=LENGTH)
  actions = np.random.RandomState(5).randint(0, 17, (T, K))
  vecs, finals = [env.gather(env.reset())], []
  for t in range(T):
    vec, reward, done, info = env.step(actions[t, env.local_slice()])
    full_vec, full_final = env.gather(vec, info['final_observation'])
    assert full_vec.dtype == torch.float32
    vecs.append(full_vec)
    finals.append(full_final)
  if rank == 0:
    shared['vec'] = np.stack([v.numpy() for v in vecs])
    shared['final'] = np.stack([f.numpy() for f in finals])
  dist.destroy_process_group()


def test_two_rank_symbolic_shards_equal_one_batch():
  from tests.test_symbolic_obs import SimtSymbolicEnv
  ctx = mp.get_context('spawn')  # never fork a multi-threaded pytest process
  manager = ctx.Manager()
  out = manager.dict()
  port = _free_port()
  procs = [ctx.Process(target=_worker, args=(r, 2, port, out)) for r in range(2)]
  for p in procs:
    p.start()
  for p in procs:
    p.join(300)
    assert p.exitcode == 0
  ref = SimtSymbolicEnv(num_envs=K, seed=11, auto_reset=True, length=LENGTH, final_obs=True)
  actions = np.random.RandomState(5).randint(0, 17, (T, K))
  vecs, finals, dones = [ref.reset().copy()], [], []
  for t in range(T):
    vec, _, done = ref.step(actions[t])
    vecs.append(vec.copy()); finals.append(ref.final_symbolic.copy()); dones.append(done.copy())
  assert (np.stack(vecs).view(np.uint32) == out['vec'].view(np.uint32)).all()
  assert (np.stack(finals).view(np.uint32) == out['final'].view(np.uint32)).all()
  assert np.stack(dones).any(), 'the run should cross at least one auto-reset'
