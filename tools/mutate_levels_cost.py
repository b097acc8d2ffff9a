"""tools/mutate_levels_cost.py -- what level mutation (Env.mutate_levels) costs on one GPU, against the torch loop a
caller would write without it.

For area 64 x 64 and 256 x 256, 256 and 4,096 children, 20 and 200 edits, on a table of as many entries with its
cache filled (the children are a permutation of the table, the parents drawn at random from it):

1. `kernel`: device time of one cr_mutate_levels call (k_mutate and authoring's four launches), CUDA events around
   the call, `--reps` calls on a warmed handle, the mean of all but the first.
2. `env`: host wall clock of Env.mutate_levels, which adds the host checks and reads the status words back.
3. `torch`: the same number of edits as a caller's torch loop: level_worlds, then per edit a gather of the drawn
   cells, the rules of the ops as torch.where and a scatter back, for all children at once, then author_levels.
   Its draws come from torch's generator (made ahead, outside the loop's per-edit launches), so its children differ
   from the kernel's; only the time is compared.  Host wall clock ending in a device synchronise, `--torch-reps`
   calls, the mean of all but the first.

Prints the card's name, power limit and clocks, then one JSON line.  bench.py is not timed here: no step code
changes with level mutation.

    python tools/mutate_levels_cost.py [--reps 6] [--torch-reps 3]
"""
import argparse
import json
import pathlib
import sys
import time

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from tools.level_sampler_cost import card  # noqa: E402

AREAS = ((64, 64), (256, 256))
COUNTS = (256, 4096)
EDITS = (20, 200)
WEIGHTS = {'cow': 2, 'zombie': 2, 'skeleton': 1, 'remove': 1, 'stone': 2, 'tree': 2, 'water': 1, 'lava': 1,
           'grass': 2, 'sand': 1, 'path': 1, 'table': 1}


def torch_loop(env, parents, children, edits, gen):
  """The caller's loop: level_worlds -> per-edit torch ops for every child at once -> author_levels."""
  import torch
  from crafter_b200.env import MUTATE_OPS, mutate_weights
  dev = env.device
  W, H = env._area
  k, nc = len(children), W * H
  start = (W // 2) * H + H // 2
  w = env.level_worlds(parents)
  m = w['materials'].reshape(k, nc).long()
  c = w['creatures'].reshape(k, nc).long()
  count = (c != 0).sum(1)
  cell = torch.randint(0, nc - 1, (edits, k), generator=gen, device=dev)
  cell += cell >= start
  weights = torch.tensor(mutate_weights(WEIGHTS), dtype=torch.float32, device=dev)
  op = torch.multinomial(weights, edits * k, replacement=True, generator=gen).view(edits, k)
  walk = torch.zeros(len(MUTATE_OPS), dtype=torch.bool, device=dev)
  walk[[2, 4, 5]] = True  # grass, path, sand
  rows = torch.arange(k, device=dev)
  cap = env._capacity - 2
  for j in range(edits):
    cj, oj = cell[j], op[j]
    mat, cre = m[rows, cj], c[rows, cj]
    new_mat = torch.where(oj < 12, oj + 1, mat)
    drop = (oj < 12) & (cre != 0) & ~walk[new_mat]
    place = (oj >= 12) & (oj < 15) & walk[mat] & ((cre != 0) | (count < cap))
    gone = drop | ((oj == 15) & (cre != 0))
    new_cre = torch.where(gone, 0, torch.where(place, oj - 11, cre))
    count += (place & (cre == 0)).long() - gone.long()
    m[rows, cj] = new_mat
    c[rows, cj] = new_cre
  env.author_levels(children, m.view(k, W, H), c.view(k, W, H))


def measure(area, count, edits, args, device):
  import ctypes

  import numpy as np
  import torch
  import crafter_b200
  from crafter_b200 import _cabi
  from crafter_b200.env import MUTATE_OPS, mutate_weights
  rs = np.random.RandomState(count + edits)
  env = crafter_b200.Env(num_envs=8, seed=0, auto_reset=True, device=device, area=area)
  env.set_level_table(rs.randint(0, 2 ** 31 - 1, count))
  env.set_level_cache()
  parents = torch.as_tensor(rs.randint(0, count, count), dtype=torch.int32, device=device)
  children = torch.as_tensor(rs.permutation(count), dtype=torch.int32, device=device)
  worlds = torch.empty(count, area[0] * area[1], dtype=torch.uint8, device=device)
  status = torch.empty(count, dtype=torch.int32, device=device)
  host_w = (ctypes.c_uint32 * len(MUTATE_OPS))(*mutate_weights(WEIGHTS))
  stream = torch.cuda.current_stream(device)
  times = []
  for rep in range(args.reps):
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record(stream)
    _cabi.check(env._lib.cr_mutate_levels(env._handle, parents.data_ptr(), children.data_ptr(), count, edits, host_w,
                                          rep, worlds.data_ptr(), status.data_ptr(), stream.cuda_stream))
    t1.record(stream)
    torch.cuda.synchronize(device)
    assert int(status.abs().sum()) == 0
    times.append(t0.elapsed_time(t1))
  kernel = sum(times[1:]) / max(1, len(times) - 1)
  wall = []
  for rep in range(args.reps):
    torch.cuda.synchronize(device)
    t = time.perf_counter()
    env.mutate_levels(parents, children, edits, 1000 + rep, WEIGHTS)
    torch.cuda.synchronize(device)
    wall.append(1000 * (time.perf_counter() - t))
  loop = []
  gen = torch.Generator(device=device).manual_seed(5)
  for _ in range(args.torch_reps):
    torch.cuda.synchronize(device)
    t = time.perf_counter()
    torch_loop(env, parents, children, edits, gen)
    torch.cuda.synchronize(device)
    loop.append(1000 * (time.perf_counter() - t))
  env.close()
  mean = lambda xs: sum(xs[1:]) / max(1, len(xs) - 1)
  return {'area': list(area), 'children': count, 'edits': edits, 'kernel_ms': round(kernel, 3),
          'env_ms': round(mean(wall), 3), 'torch_ms': round(mean(loop), 3),
          'torch_over_kernel': round(mean(loop) / kernel, 1), 'torch_over_env': round(mean(loop) / mean(wall), 1)}


def main():
  ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
  ap.add_argument('--reps', type=int, default=6)
  ap.add_argument('--torch-reps', type=int, default=3)
  args = ap.parse_args()
  import torch
  if not torch.cuda.is_available():
    raise SystemExit('mutate_levels_cost.py needs a CUDA device')
  device = torch.device('cuda', 0)
  print('card:', card())
  out = []
  for area in AREAS:
    for count in COUNTS:
      for edits in EDITS:
        r = measure(area, count, edits, args, device)
        print(r, flush=True)
        out.append(r)
  print(json.dumps({'card': card(), 'mutate_levels': out}))


if __name__ == '__main__':
  main()
