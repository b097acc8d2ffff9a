"""tools/level_sampler_cost.py -- what choosing levels costs on one GPU, from outside the step and inside it.

1. `bench.py` at a parent tree (`--parent DIR`, a checkout of the commit before the level sampler with its library
   built) and at this tree, alternated `--ab-reps` times each: the default workload's env-steps/s, whose only
   change is one compare of the already-loaded level in k_seed.
2. Steady-state env-steps/s at 4096 envs (bench.py's default workload, auto-reset, after a 1,000-step pre-roll)
   for frames (observation='rgb') and symbolic vectors, in five patterns:
     plain          step() only;
     set_levels     step(), then Env.set_levels on the envs that finished, drawn from 200 world seeds on the
                    host's side of the step (tools/levels_cost.py's pattern: a second world generation and a
                    host read per step);
     sampled        every env sampled (Env.sample_levels) from the same 200 seeds, uniform weights: step() only;
     sampled_plr    as `sampled`, with Env.set_level_weights of a fresh device tensor before every step (the
                    prioritized-level-replay loop: torch's cumsum and copies, no launch of the library);
     sampled_plr_1m as `sampled_plr` with a table of 2**20 seeds.
   Host wall clock over `--steps` steps ending in a device synchronise.  The patterns are timed alternately,
   `--reps` windows each, on envs of the same seed.

Prints the card's name, power limit and clocks, then one JSON line.

    python tools/level_sampler_cost.py [--parent DIR] [--ab-reps 3] [--steps 500] [--reps 3]
"""
import argparse
import json
import pathlib
import subprocess
import sys
import time

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import bench  # noqa: E402
from tools.levels_cost import ab  # noqa: E402

PATTERNS = ('plain', 'set_levels', 'sampled', 'sampled_plr', 'sampled_plr_1m')


def card(index=0):
  return subprocess.run(['nvidia-smi', f'--id={index}', '--query-gpu=name,power.limit,clocks.max.sm,clocks.sm',
                         '--format=csv,noheader'], capture_output=True, text=True, timeout=60).stdout.strip()


def patterns(observation, args, device):
  import torch
  import crafter_b200
  from crafter_b200 import state as state_lib
  kwargs = bench.env_kwargs(bench.CONFIGS['default'])
  B = kwargs['num_envs']
  T = 512
  gen = torch.Generator(device=device).manual_seed(1234)
  actions = torch.randint(0, 17, (T, B), generator=gen, device=device, dtype=torch.int32)
  pool = torch.randint(0, 2 ** 31 - 1, (200,), generator=gen, device=device, dtype=torch.int32)
  big = torch.randint(0, 2 ** 31 - 1, (2 ** 20,), generator=gen, device=device, dtype=torch.int32)
  envs = {p: crafter_b200.Env(seed=0, auto_reset=True, device=device, observation=observation, **kwargs)
          for p in PATTERNS}
  draws = torch.Generator(device=device).manual_seed(7)
  # 16 weight vectors per table, made ahead: the timed loop pays for set_level_weights, not for inventing priorities
  weights = {'sampled_plr': torch.randint(1, 2 ** 16, (16, 200), generator=gen, device=device, dtype=torch.int64),
             'sampled_plr_1m': torch.randint(1, 2 ** 11, (16, 2 ** 20), generator=gen, device=device, dtype=torch.int64)}

  def start(env, p):
    if p.startswith('sampled'):
      env.set_level_table(big if p == 'sampled_plr_1m' else pool)
      env.sample_levels()

  def one_step(env, p, t):
    if p in weights:
      env.set_level_weights(weights[p][t % 16])
    done = env.step(actions[t % T])[2]
    if p == 'set_levels':
      env.set_levels(pool[torch.randint(0, len(pool), (B,), generator=draws, device=device)], done)

  pos = args.preroll + args.warmup
  for p in PATTERNS:
    envs[p].reset()
    for t in range(args.preroll):
      one_step(envs[p], 'plain', t)  # the pre-roll itself is plain
    start(envs[p], p)
    for t in range(args.preroll, pos):
      one_step(envs[p], p, t)
  torch.cuda.synchronize(device)
  rates = {p: [] for p in PATTERNS}
  for _ in range(args.reps):
    for p in PATTERNS:
      torch.cuda.synchronize(device)
      t0 = time.perf_counter()
      for k in range(args.steps):
        one_step(envs[p], p, pos + k)
      torch.cuda.synchronize(device)
      rates[p].append(B * args.steps / (time.perf_counter() - t0))
    pos += args.steps
  started = {p: int(envs[p].state['pstate'][:, state_lib.PS['episode']].sum()) for p in PATTERNS}
  for p, env in envs.items():
    env.check_errors()
    env.close()
  mean = {p: sum(v) / len(v) for p, v in rates.items()}
  return {'env_steps_per_sec': {p: [round(x) for x in v] for p, v in rates.items()},
          'us_per_step': {p: round(1e6 * B / mean[p], 1) for p in PATTERNS},
          'over_plain': {p: round(mean[p] / mean['plain'], 4) for p in PATTERNS}, 'episodes_started': started}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--parent', help='a tree of the commit before the level sampler, its library built (bench.py A/B)')
  ap.add_argument('--ab-reps', type=int, default=3)
  ap.add_argument('--bench-steps', type=int, default=2000)
  ap.add_argument('--bench-warmup', type=int, default=200)
  ap.add_argument('--steps', type=int, default=500)
  ap.add_argument('--warmup', type=int, default=50)
  ap.add_argument('--preroll', type=int, default=1000)
  ap.add_argument('--reps', type=int, default=3)
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
  out.update(steps=args.steps, warmup=args.warmup, preroll=args.preroll, reps=args.reps, patterns={})
  for observation in ('rgb', 'symbolic'):
    out['patterns'][observation] = patterns(observation, args, device)
    print(observation, json.dumps(out['patterns'][observation]), flush=True)
  print(json.dumps(out))


if __name__ == '__main__':
  main()
