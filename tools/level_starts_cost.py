"""tools/level_starts_cost.py -- what level starts (Env.set_level_starts) cost on one GPU.

1. `bench.py` at a parent tree (`--parent DIR`, a checkout of the commit before the starts with its library built) and
   at this tree, alternated `--ab-reps` times each: the default path, which gains one null test in k_seed and one in
   k_install.
2. Overhead: steady-state us per step of bench.py's three workloads (default, area256, view15) x observation 'rgb' /
   'semantic' / 'symbolic', auto-reset, every env sampled from 200 cached world seeds, without starts (`none`) and
   with starts registered, every record 0 (`zero`).  The two runs play the same episodes, so any difference is the
   cost of the start path itself: an 80-byte copy per decided seed and one barrier per installed episode.
3. Workload: the same batch with starts on half of the entries (`starts`: within 3 cells of the centre, random
   inventories and vitals).  Those episodes play differently (other vitals, other deaths), so the resets per step are
   reported beside the step time, so that a slower step is not misread as overhead.
Host wall clock over `--steps` steps ending in a device synchronise; the patterns are timed alternately, `--reps`
windows each, on envs of the same seed after a `--preroll`-step pre-roll.

Prints the card's name, power limit and clocks, then one JSON line.

    python tools/level_starts_cost.py [--parent DIR] [--ab-reps 3] [--steps 300] [--reps 3]
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

PATTERNS = ('none', 'zero', 'starts')
WORKLOADS = ('default', 'area256', 'view15')
OBSERVATIONS = ('rgb', 'semantic', 'symbolic')


def start_table(n, area):
  import numpy as np
  from crafter_b200 import rules
  from crafter_b200.env import START_WORDS, level_start
  rs = np.random.RandomState(9)
  W, H = area
  rows = np.zeros((n, START_WORDS), np.int32)
  for r in np.flatnonzero(rs.rand(n) < 0.5):
    inv = {name: int(rs.randint(0, 10)) for name in rules.ITEMS if rs.rand() < 0.4}
    inv['health'] = int(rs.randint(1, 10))
    rows[r] = level_start(inv, (W // 2 + rs.randint(-3, 4), H // 2 + rs.randint(-3, 4)),
                          ('left', 'right', 'up', 'down')[rs.randint(0, 4)], area)
  return rows


def make(workload, observation, device, table, pattern):
  import numpy as np
  import crafter_b200
  from crafter_b200.env import START_WORDS
  cfg = bench.CONFIGS[workload]
  env = crafter_b200.Env(seed=0, auto_reset=True, device=device, observation=observation, **bench.env_kwargs(cfg))
  env.set_level_table(table)
  env.set_level_cache()
  if pattern == 'zero':
    env.set_level_starts(np.zeros((len(table), START_WORDS), np.int32))
  elif pattern == 'starts':
    env.set_level_starts(start_table(len(table), cfg['area']))
  env.sample_levels()
  env.reset()
  return env


def rates(workload, observation, args, device, table):
  import torch
  B = bench.CONFIGS[workload]['num_envs']
  T = 256
  gen = torch.Generator(device=device).manual_seed(1234)
  actions = torch.randint(0, 17, (T, B), generator=gen, device=device, dtype=torch.int32)
  envs = {p: make(workload, observation, device, table, p) for p in PATTERNS}
  for env in envs.values():
    for t in range(args.preroll):
      env.step(actions[t % T])
  pos = args.preroll
  torch.cuda.synchronize(device)
  got = {p: [] for p in PATTERNS}
  resets = {p: torch.zeros((), dtype=torch.int64, device=device) for p in PATTERNS}
  for _ in range(args.reps):
    for p in PATTERNS:
      env = envs[p]
      torch.cuda.synchronize(device)
      t0 = time.perf_counter()
      for k in range(args.steps):
        env.step(actions[(pos + k) % T])
      torch.cuda.synchronize(device)
      got[p].append(1e6 * (time.perf_counter() - t0) / args.steps)
    pos += args.steps
  for p, env in envs.items():  # resets per step, counted in an untimed window of the same length
    for k in range(args.steps):
      _, _, done, _ = env.step(actions[(pos + k) % T])
      resets[p] += done.sum()
  out_resets = {p: round(int(v) / args.steps, 2) for p, v in resets.items()}
  flags = {p: env.error_flags() for p, env in envs.items()}  # 8 where a start cell was not walkable (the 'starts' batch)
  for env in envs.values():
    env.close()
  mean = {p: sum(v) / len(v) for p, v in got.items()}
  return {'us_per_step': {p: [round(x, 1) for x in v] for p, v in got.items()},
          'over_none': {p: round(mean[p] / mean['none'], 4) for p in PATTERNS},
          'resets_per_step': out_resets, 'error_flags': flags}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--parent', help='a tree of the commit before the starts, its library built (bench.py A/B)')
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
  out.update(steps=args.steps, preroll=args.preroll, reps=args.reps, patterns={})
  for workload in args.workloads.split(','):
    for observation in OBSERVATIONS:
      key = f'{workload}/{observation}'
      out['patterns'][key] = rates(workload, observation, args, device, table)
      print(key, json.dumps(out['patterns'][key]), flush=True)
  print(json.dumps(out))


if __name__ == '__main__':
  main()
