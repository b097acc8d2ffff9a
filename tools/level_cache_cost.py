"""tools/level_cache_cost.py -- what the level cache (Env.set_level_cache) buys and costs on one GPU.

1. `bench.py` at a parent tree (`--parent DIR`, a checkout of the commit before the level cache with its library
   built) and at this tree, alternated `--ab-reps` times each: the default path, which gains one null-pointer test
   in k_seed, k_wg_mat and k_wg_obj.
2. Steady-state env-steps/s of bench.py's three workloads (default, area256, view15) x observation 'rgb' /
   'semantic' / 'symbolic', auto-reset, after a `--preroll`-step plain pre-roll, in five patterns:
     plain         step() only;
     sampled       every env sampled (Env.sample_levels) from 200 world seeds, uniform weights, no cache;
     cached        as `sampled`, with Env.set_level_cache();
     cached_64k    as `cached` with a table of 2**16 seeds;
     cached_plr    as `cached`, with Env.set_level_weights of a fresh device tensor before every step.
   Host wall clock over `--steps` steps ending in a device synchronise; the patterns are timed alternately,
   `--reps` windows each, on envs of the same seed.
3. In-graph kernel times (CRAFTER_B200_TIMING=2: events as nodes of the step graph) of plain, sampled and cached
   at each workload and observation: k_seed (ahead), k_wg_mat, k_wg_obj, install.
4. The fill: device time per world of Env.set_level_cache over 2**16 seeds, and the bytes per world.

Prints the card's name, power limit and clocks, then one JSON line.

    python tools/level_cache_cost.py [--parent DIR] [--ab-reps 3] [--steps 300] [--reps 3]
"""
import argparse
import json
import os
import pathlib
import sys
import time

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import bench  # noqa: E402
from tools.level_sampler_cost import card  # noqa: E402
from tools.levels_cost import ab  # noqa: E402

PATTERNS = ('plain', 'sampled', 'cached', 'cached_64k', 'cached_plr')
WORKLOADS = ('default', 'area256', 'view15')
OBSERVATIONS = ('rgb', 'semantic', 'symbolic')
TIMING_KEYS = ('update', 'install', 'render', 'seed', 'wg_mat', 'wg_obj', 'seed_ahead', 'balance')  # cr_timing order


def make(workload, observation, device):
  import crafter_b200
  env = crafter_b200.Env(seed=0, auto_reset=True, device=device, observation=observation,
                         **bench.env_kwargs(bench.CONFIGS[workload]))
  env.reset()
  return env


def start(env, pattern, tables):
  if pattern == 'plain':
    return
  env.set_level_table(tables['64k' if pattern == 'cached_64k' else '200'])
  if pattern != 'sampled':
    env.set_level_cache()
  env.sample_levels()


def rates(workload, observation, args, device, tables, weights):
  import torch
  B = bench.CONFIGS[workload]['num_envs']
  T = 256
  gen = torch.Generator(device=device).manual_seed(1234)
  actions = torch.randint(0, 17, (T, B), generator=gen, device=device, dtype=torch.int32)
  envs = {p: make(workload, observation, device) for p in PATTERNS}

  def one_step(env, p, t):
    if p == 'cached_plr':
      env.set_level_weights(weights[t % 16])
    env.step(actions[t % T])

  pos = args.preroll + args.warmup
  for p, env in envs.items():
    for t in range(args.preroll):
      one_step(env, 'plain', t)
    start(env, p, tables)
    for t in range(args.preroll, pos):
      one_step(env, p, t)
  torch.cuda.synchronize(device)
  got = {p: [] for p in PATTERNS}
  for _ in range(args.reps):
    for p in PATTERNS:
      torch.cuda.synchronize(device)
      t0 = time.perf_counter()
      for k in range(args.steps):
        one_step(envs[p], p, pos + k)
      torch.cuda.synchronize(device)
      got[p].append(B * args.steps / (time.perf_counter() - t0))
    pos += args.steps
  for env in envs.values():
    env.check_errors()
    env.close()
  mean = {p: sum(v) / len(v) for p, v in got.items()}
  return {'env_steps_per_sec': {p: [round(x) for x in v] for p, v in got.items()},
          'us_per_step': {p: round(1e6 * B / mean[p], 1) for p in PATTERNS},
          'over_plain': {p: round(mean[p] / mean['plain'], 4) for p in PATTERNS}}


def kernel_times(workload, observation, args, device, tables):
  """Mean in-graph device us per step of the step's kernels, plain / sampled / cached (CRAFTER_B200_TIMING=2)."""
  import ctypes
  import torch
  B = bench.CONFIGS[workload]['num_envs']
  gen = torch.Generator(device=device).manual_seed(99)
  out = {}
  os.environ['CRAFTER_B200_TIMING'] = '2'
  try:
    for p in ('plain', 'sampled', 'cached'):
      env = make(workload, observation, device)
      for t in range(args.preroll):
        env.step(torch.randint(0, 17, (B,), generator=gen, device=device, dtype=torch.int32))
      start(env, p, tables)
      for t in range(args.warmup):
        env.step(torch.randint(0, 17, (B,), generator=gen, device=device, dtype=torch.int32))
      ms = (ctypes.c_double * len(TIMING_KEYS))()
      env._lib.cr_timing(env._handle, ms)  # drop what was accumulated so far
      for t in range(args.steps):
        env.step(torch.randint(0, 17, (B,), generator=gen, device=device, dtype=torch.int32))
      n = env._lib.cr_timing(env._handle, ms)
      out[p] = dict({k: round(1000 * ms[i], 1) for i, k in enumerate(TIMING_KEYS)}, steps=int(n))
      env.close()
  finally:
    del os.environ['CRAFTER_B200_TIMING']
  return out


def fill_cost(workload, device, tables):
  import torch
  import crafter_b200
  env = crafter_b200.Env(seed=0, auto_reset=True, device=device, **bench.env_kwargs(bench.CONFIGS[workload]))
  env.set_level_table(tables['64k'])
  torch.cuda.synchronize(device)
  t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  t0.record()
  env.set_level_cache()
  t1.record()
  torch.cuda.synchronize(device)
  n = len(tables['64k'])
  info = env.level_cache
  env.close()
  return {'worlds': n, 'us_per_world': round(1000 * t0.elapsed_time(t1) / n, 3),
          'bytes_per_world': info['bytes_per_world'], 'bytes': info['bytes']}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--parent', help='a tree of the commit before the level cache, its library built (bench.py A/B)')
  ap.add_argument('--ab-reps', type=int, default=3)
  ap.add_argument('--bench-steps', type=int, default=2000)
  ap.add_argument('--bench-warmup', type=int, default=200)
  ap.add_argument('--steps', type=int, default=300)
  ap.add_argument('--warmup', type=int, default=50)
  ap.add_argument('--preroll', type=int, default=1000)
  ap.add_argument('--reps', type=int, default=3)
  ap.add_argument('--workloads', default=','.join(WORKLOADS))
  args = ap.parse_args()
  gpu = card(0)
  print('card, power limit, max SM clock, SM clock now:', gpu, flush=True)
  out = {'gpu_power_limit_clocks': gpu}
  if args.parent:
    out['bench_ab'] = ab(pathlib.Path(args.parent).resolve(), args.ab_reps, args.bench_steps, args.bench_warmup)
    print('bench_ab', json.dumps(out['bench_ab']), flush=True)
  import torch
  device = torch.device('cuda', 0)
  torch.cuda.set_device(device)
  gen = torch.Generator(device=device).manual_seed(1234)
  tables = {'200': torch.randint(0, 2 ** 31 - 1, (200,), generator=gen, device=device, dtype=torch.int32),
            '64k': torch.randint(0, 2 ** 31 - 1, (2 ** 16,), generator=gen, device=device, dtype=torch.int32)}
  weights = torch.randint(1, 2 ** 16, (16, 200), generator=gen, device=device, dtype=torch.int64)
  out.update(steps=args.steps, warmup=args.warmup, preroll=args.preroll, reps=args.reps, patterns={}, kernels={},
             fill={})
  for workload in args.workloads.split(','):
    out['fill'][workload] = fill_cost(workload, device, tables)
    print(workload, 'fill', json.dumps(out['fill'][workload]), flush=True)
    for observation in OBSERVATIONS:
      key = f'{workload}/{observation}'
      out['patterns'][key] = rates(workload, observation, args, device, tables, weights)
      print(key, json.dumps(out['patterns'][key]), flush=True)
      out['kernels'][key] = kernel_times(workload, observation, args, device, tables)
      print(key, 'kernels', json.dumps(out['kernels'][key]), flush=True)
  print(json.dumps(out))


if __name__ == '__main__':
  main()
