"""tools/level_stats_cost.py -- what per-level episode statistics (Env.set_level_stats) cost on one GPU.

1. `bench.py` at a parent tree (`--parent DIR`, a checkout of the commit before the statistics with its library
   built) and at this tree, alternated `--ab-reps` times each: the default path, which gains one null test in k_seed
   and one in the tick's done branch.
2. Steady-state us per step of bench.py's three workloads (default, area256, view15) x observation 'rgb' /
   'semantic' / 'symbolic', auto-reset, every env sampled from 200 cached world seeds, in six patterns:
     cached          no statistics;
     stats           Env.set_level_stats();
     plr_1, plr_10   stats, and every 1 / 10 steps the whole loop a caller runs: level_stats(), level_scores(),
                     integer weights from the scores, set_level_weights(), clear_level_stats() -- no host read;
     weights_1, weights_10   the same cadence of set_level_weights without statistics (weights from a fixed pool).
   Host wall clock over `--steps` steps ending in a device synchronise; the patterns are timed alternately, `--reps`
   windows each, on envs of the same seed after a `--preroll`-step pre-roll.

Prints the card's name, power limit and clocks, then one JSON line.

    python tools/level_stats_cost.py [--parent DIR] [--ab-reps 3] [--steps 300] [--reps 3]
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

PATTERNS = ('cached', 'stats', 'plr_1', 'plr_10', 'weights_1', 'weights_10')
WORKLOADS = ('default', 'area256', 'view15')
OBSERVATIONS = ('rgb', 'semantic', 'symbolic')


def make(workload, observation, device, table, stats):
  import crafter_b200
  env = crafter_b200.Env(seed=0, auto_reset=True, device=device, observation=observation,
                         **bench.env_kwargs(bench.CONFIGS[workload]))
  env.set_level_table(table)
  env.set_level_cache()
  if stats:
    env.set_level_stats()
  env.sample_levels()
  env.reset()
  return env


def plr_weights(env):
  """The caller's side of a PLR-style loop: scores from the counts, lower scores weighted up, then a new window."""
  import torch
  from crafter_b200.env import level_scores
  _, score = level_scores(env.level_stats())
  w = ((101 - torch.nan_to_num(score, nan=0.0)) * 2 ** 16).round().to(torch.int64)  # total < 2**32 for 200 seeds
  env.set_level_weights(w)
  env.clear_level_stats()


def rates(workload, observation, args, device, table, pool):
  import torch
  B = bench.CONFIGS[workload]['num_envs']
  T = 256
  gen = torch.Generator(device=device).manual_seed(1234)
  actions = torch.randint(0, 17, (T, B), generator=gen, device=device, dtype=torch.int32)
  envs = {p: make(workload, observation, device, table, p in ('stats', 'plr_1', 'plr_10')) for p in PATTERNS}

  def one_step(env, p, t):
    if p.startswith('plr_') and t % int(p[4:]) == 0:
      plr_weights(env)
    elif p.startswith('weights_') and t % int(p[8:]) == 0:
      env.set_level_weights(pool[t % len(pool)])
    env.step(actions[t % T])

  for p, env in envs.items():
    for t in range(args.preroll):
      one_step(env, p, t)
  pos = args.preroll
  torch.cuda.synchronize(device)
  got = {p: [] for p in PATTERNS}
  for _ in range(args.reps):
    for p in PATTERNS:
      torch.cuda.synchronize(device)
      t0 = time.perf_counter()
      for k in range(args.steps):
        one_step(envs[p], p, pos + k)
      torch.cuda.synchronize(device)
      got[p].append(1e6 * (time.perf_counter() - t0) / args.steps)
    pos += args.steps
  counted = int(envs['stats'].level_stats()['episodes'].sum())
  for env in envs.values():
    env.check_errors()
    env.close()
  mean = {p: sum(v) / len(v) for p, v in got.items()}
  return {'us_per_step': {p: [round(x, 1) for x in v] for p, v in got.items()},
          'over_cached': {p: round(mean[p] / mean['cached'], 4) for p in PATTERNS},
          'episodes_counted_by_stats': counted}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--parent', help='a tree of the commit before the statistics, its library built (bench.py A/B)')
  ap.add_argument('--ab-reps', type=int, default=3)
  ap.add_argument('--bench-steps', type=int, default=2000)
  ap.add_argument('--bench-warmup', type=int, default=200)
  ap.add_argument('--steps', type=int, default=300)
  ap.add_argument('--preroll', type=int, default=600)
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
  table = torch.randint(0, 2 ** 31 - 1, (200,), generator=gen, device=device, dtype=torch.int32)
  pool = torch.randint(1, 2 ** 16, (16, 200), generator=gen, device=device, dtype=torch.int64)
  out.update(steps=args.steps, preroll=args.preroll, reps=args.reps, patterns={})
  for workload in args.workloads.split(','):
    for observation in OBSERVATIONS:
      key = f'{workload}/{observation}'
      out['patterns'][key] = rates(workload, observation, args, device, table, pool)
      print(key, json.dumps(out['patterns'][key]), flush=True)
  print(json.dumps(out))


if __name__ == '__main__':
  main()
