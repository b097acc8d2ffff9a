"""Batch sharding across the GPUs of one node: one process per GPU, no collective on the step path.

Environments are independent (the reference builds one `World` per `Env`, env.py:40) and every
random draw is keyed by (base seed + global env index, episode, ...), so rank r simply owns the
global envs [r * n, (r + 1) * n) and the union over ranks equals one big batch bit for bit,
whatever the number of GPUs.  `gather()` is the only collective: an opt-in NCCL all-gather of
obs / reward / done over NVLink for callers that want whole-batch tensors on every rank.
"""
import os

import torch
import torch.distributed as dist


def shard_of(total_envs, rank, world):
  """Contiguous shard [start, start + count) of `total_envs` global env indices for `rank`."""
  if total_envs % world:
    raise ValueError(f'num_envs={total_envs} is not divisible by world size {world}')
  count = total_envs // world
  return rank * count, count


class ShardedEnv:
  """`crafter_b200.Env` over the whole job: `num_envs` is the GLOBAL batch; this process steps its
  own shard on `cuda:LOCAL_RANK`.  reset()/step() return the local shard's tensors.  Keyword arguments go to
  the env unchanged (e.g. `observation='semantic'` or `'symbolic'`: `gather` takes windows and float32 vectors
  as it takes frames).  The env's other methods pass through: set_levels, sample_levels and pin_levels take the
  LOCAL shard's levels, entries and mask; set_level_table / set_level_weights take the same table on every rank,
  and author_levels the same worlds on every rank, and since the draw is keyed by the global env index the shards
  then play what one big batch plays.  mutate_levels makes the same children on every rank when every rank makes
  the same call: a child is a function of its parent's world, the key, its entry, the edits and the weights alone,
  so no bytes need to be broadcast.  level_stats gives the LOCAL shard's counts; they are integers, so their sum
  over the ranks (an all-reduce) is exactly what one big batch counts.  set_level_goals takes the same goals on
  every rank, and set_level_starts, like the goals, the same starts on every rank."""

  def __init__(self, num_envs, seed=0, env_factory=None, **kwargs):
    self.rank = dist.get_rank() if dist.is_initialized() else int(os.environ.get('RANK', 0))
    self.world = dist.get_world_size() if dist.is_initialized() else int(os.environ.get('WORLD_SIZE', 1))
    self.global_num_envs = int(num_envs)
    self.offset, self.local_num_envs = shard_of(num_envs, self.rank, self.world)
    if env_factory is None:
      from .env import Env as env_factory
      kwargs.setdefault('device', torch.device('cuda', int(os.environ.get('LOCAL_RANK', 0))))
    self.env = env_factory(num_envs=self.local_num_envs, seed=seed, env_offset=self.offset, **kwargs)

  def __getattr__(self, name):
    return getattr(self.env, name)

  def reset(self, mask=None, levels=None):
    """`mask` and `levels` (see Env.reset / Env.set_levels) are the LOCAL shard's, like actions."""
    if levels is None:  # env factories without levels keep working
      return self.env.reset(mask)
    return self.env.reset(mask, levels)

  def step(self, actions):
    """`actions` are the LOCAL shard's actions, shape (local_num_envs,)."""
    return self.env.step(actions)

  def local_slice(self):
    return slice(self.offset, self.offset + self.local_num_envs)

  def gather(self, *tensors):
    """All-gather local tensors along dim 0 into whole-batch tensors on every rank (opt-in; at
    32768 envs the obs gather moves 352 MB per step per GPU, so keep it off the hot path)."""
    out = []
    for t in tensors:
      t = t.contiguous()
      if self.world == 1:
        out.append(t)
        continue
      flags = t.dtype == torch.bool
      src = t.to(torch.uint8) if flags else t
      full = torch.empty((self.global_num_envs,) + tuple(src.shape[1:]), dtype=src.dtype,
                         device=src.device)
      dist.all_gather_into_tensor(full, src)
      out.append(full.to(torch.bool) if flags else full)
    return out[0] if len(out) == 1 else tuple(out)

  def gather_async(self, tensor):
    """The same all-gather, off the step path: `tensor` (e.g. the obs view, which the next step()
    overwrites) is snapshotted on the current stream, the collective runs on a side stream while the
    caller keeps stepping, and the returned handle's `.wait()` makes the current stream wait for the
    whole-batch tensor and returns it.  Two snapshots / results are kept, so one gather may be in
    flight while the next is issued (wait on a handle before issuing the one after next)."""
    if self.world == 1:
      return _Ready(tensor)
    if not hasattr(self, '_ga'):
      self._ga = dict(stream=torch.cuda.Stream(tensor.device), slot=0, bufs={})
    ga = self._ga
    key = (tuple(tensor.shape), tensor.dtype, ga['slot'])
    ga['slot'] ^= 1
    if key not in ga['bufs']:
      ga['bufs'][key] = (torch.empty_like(tensor), torch.empty((self.global_num_envs,) + tuple(tensor.shape[1:]),
                                                              dtype=tensor.dtype, device=tensor.device))
    snap, full = ga['bufs'][key]
    snap.copy_(tensor)
    ga['stream'].wait_stream(torch.cuda.current_stream(tensor.device))
    with torch.cuda.stream(ga['stream']):
      dist.all_gather_into_tensor(full, snap)
      done = torch.cuda.Event()
      done.record(ga['stream'])
    return _Pending(full, done)


class _Ready:
  def __init__(self, tensor):
    self._t = tensor

  def wait(self):
    return self._t


class _Pending:
  def __init__(self, tensor, event):
    self._t, self._e = tensor, event

  def wait(self):
    torch.cuda.current_stream(self._t.device).wait_event(self._e)
    return self._t
