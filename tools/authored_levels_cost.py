"""tools/authored_levels_cost.py -- what authored levels and pinning (Env.author_levels, Env.pin_levels) cost on one
GPU.

1. `bench.py` at a parent tree (`--parent DIR`, a checkout of the commit before authored levels with its library
   built) and at this tree, alternated `--ab-reps` times each: the default path, which gains one compare in k_seed.
2. Authoring: device time per world of cr_author_levels (check, copy, creature pass, tag) at area 64 x 64 and
   256 x 256, for 1,024 and 65,536 worlds of grass with a creature on every 97th cell, into a cache registered
   without a fill (CUDA events around the call; `--author-reps` calls, the mean of all but the first).
3. An evaluation suite: bench.py's three workloads x observation 'rgb' / 'semantic' / 'symbolic', auto-reset, every
   env pinned round robin over 200 cached table entries (`pinned`), against the same envs on set_levels of those
   entries' seeds (`set_levels`, every world generated).  Host wall clock over `--steps` steps ending in a device
   synchronise, the two timed alternately, `--reps` windows each; microseconds per step.

Prints the card's name, power limit and clocks, then one JSON line.

    python tools/authored_levels_cost.py [--parent DIR] [--ab-reps 3] [--steps 300] [--reps 3]
"""
import argparse
import json
import pathlib
import sys
import time

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import bench  # noqa: E402
from tools.level_sampler_cost import card  # noqa: E402
from tools.levels_cost import ab  # noqa: E402

WORKLOADS = ('default', 'area256', 'view15')
OBSERVATIONS = ('rgb', 'semantic', 'symbolic')
PATTERNS = ('pinned', 'set_levels')


def author_cost(area, count, reps, device):
  """Mean device ms of one cr_author_levels call of `count` worlds at `area`, and per world in us."""
  import torch
  import crafter_b200
  from crafter_b200 import _cabi
  env = crafter_b200.Env(num_envs=8, seed=0, auto_reset=True, device=device, area=area)
  env.set_level_table(torch.arange(count, dtype=torch.int32, device=device))
  W, H = area
  cells = W * H
  z = lambda *shape, dtype: torch.zeros(*shape, dtype=dtype, device=device)
  cache = dict(mat=z(count, cells, dtype=torch.uint8), ents=z(count, env._capacity, dtype=torch.int64),
               meta=z(count, 2, dtype=torch.int32), tag=torch.full((count,), -1, dtype=torch.int32, device=device),
               row=torch.full((8, 2), -1, dtype=torch.int32, device=device))
  _cabi.check(env._lib.cr_set_level_cache(env._handle, *(cache[k].data_ptr() for k in (
      'mat', 'ents', 'meta', 'tag', 'row')), count))
  world = torch.full((cells,), 2, dtype=torch.uint8, device=device)  # grass
  world[::97] |= 1 << 4  # a cow on every 97th cell
  world[(W // 2) * H + H // 2] = 2
  worlds = world.expand(count, cells).contiguous()
  entries = torch.arange(count, dtype=torch.int32, device=device)
  status = z(count, dtype=torch.int32)
  stream = torch.cuda.current_stream(device)
  times = []
  for _ in range(reps):
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record(stream)
    _cabi.check(env._lib.cr_author_levels(env._handle, entries.data_ptr(), worlds.data_ptr(), count,
                                          status.data_ptr(), stream.cuda_stream))
    t1.record(stream)
    torch.cuda.synchronize(device)
    times.append(t0.elapsed_time(t1))
  assert int(status.abs().sum()) == 0 and bool((cache['meta'][:, 1] == 5).all())
  env.close()
  mean = sum(times[1:]) / max(1, len(times) - 1)
  return {'worlds': count, 'ms_per_call': round(mean, 3), 'us_per_world': round(1000 * mean / count, 4),
          'ms_first_call': round(times[0], 3)}


def suite(workload, observation, args, device, seeds):
  import torch
  import crafter_b200
  B = bench.CONFIGS[workload]['num_envs']
  T = 256
  gen = torch.Generator(device=device).manual_seed(1234)
  actions = torch.randint(0, 17, (T, B), generator=gen, device=device, dtype=torch.int32)
  entries = torch.arange(B, device=device) % len(seeds)
  envs = {}
  for p in PATTERNS:
    env = crafter_b200.Env(seed=0, auto_reset=True, device=device, observation=observation,
                           **bench.env_kwargs(bench.CONFIGS[workload]))
    if p == 'pinned':
      env.set_level_table(seeds)
      env.set_level_cache()
      env.pin_levels(entries)
    else:
      env.set_levels(seeds[entries])
    env.reset()
    for t in range(args.warmup):
      env.step(actions[t % T])
    envs[p] = env
  torch.cuda.synchronize(device)
  got = {p: [] for p in PATTERNS}
  pos = args.warmup
  for _ in range(args.reps):
    for p in PATTERNS:
      torch.cuda.synchronize(device)
      t0 = time.perf_counter()
      for k in range(args.steps):
        envs[p].step(actions[(pos + k) % T])
      torch.cuda.synchronize(device)
      got[p].append(1e6 * (time.perf_counter() - t0) / args.steps)
    pos += args.steps
  for env in envs.values():
    env.check_errors()
    env.close()
  mean = {p: sum(v) / len(v) for p, v in got.items()}
  return {'us_per_step': {p: [round(x, 1) for x in v] for p, v in got.items()},
          'mean_us_per_step': {p: round(v, 1) for p, v in mean.items()},
          'pinned_over_set_levels_time': round(mean['pinned'] / mean['set_levels'], 4)}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--parent', help='a tree of the commit before authored levels, its library built (bench.py A/B)')
  ap.add_argument('--ab-reps', type=int, default=3)
  ap.add_argument('--bench-steps', type=int, default=2000)
  ap.add_argument('--bench-warmup', type=int, default=200)
  ap.add_argument('--author-reps', type=int, default=4)
  ap.add_argument('--steps', type=int, default=300)
  ap.add_argument('--warmup', type=int, default=100)
  ap.add_argument('--reps', type=int, default=3)
  ap.add_argument('--workloads', default=','.join(WORKLOADS))
  ap.add_argument('--skip', default='', help='comma-separated parts to skip: ab, author, suite')
  args = ap.parse_args()
  skip = set(filter(None, args.skip.split(',')))
  gpu = card(0)
  print('card, power limit, max SM clock, SM clock now:', gpu, flush=True)
  out = {'gpu_power_limit_clocks': gpu}
  if args.parent and 'ab' not in skip:
    out['bench_ab'] = ab(pathlib.Path(args.parent).resolve(), args.ab_reps, args.bench_steps, args.bench_warmup)
    print('bench_ab', json.dumps(out['bench_ab']), flush=True)
  import torch
  device = torch.device('cuda', 0)
  torch.cuda.set_device(device)
  if 'author' not in skip:
    out['author'] = {}
    for area in ((64, 64), (256, 256)):
      for count in (1024, 65536):
        key = f'{area[0]}x{area[1]}/{count}'
        out['author'][key] = author_cost(area, count, args.author_reps, device)
        print('author', key, json.dumps(out['author'][key]), flush=True)
  if 'suite' not in skip:
    seeds = torch.randint(0, 2 ** 31 - 1, (200,), generator=torch.Generator(device=device).manual_seed(5),
                          device=device, dtype=torch.int32)
    out.update(steps=args.steps, warmup=args.warmup, reps=args.reps, suite={})
    for workload in args.workloads.split(','):
      for observation in OBSERVATIONS:
        key = f'{workload}/{observation}'
        out['suite'][key] = suite(workload, observation, args, device, seeds)
        print('suite', key, json.dumps(out['suite'][key]), flush=True)
  out['gpu_power_limit_clocks_end'] = card(0)
  print(json.dumps(out))


if __name__ == '__main__':
  main()
