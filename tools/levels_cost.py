"""tools/levels_cost.py -- what levels cost on one GPU.

1. `bench.py` at a parent tree (`--parent DIR`, a checkout of the commit before levels with its library built)
   and at this tree, alternated `--ab-reps` times each in this one process group: the default workload's
   env-steps/s, whose only changes are one load per generated world in k_seed and one store per finished env
   in the tick.
2. Steady-state env-steps/s at 4096 envs (bench.py's default workload, auto-reset, after a 1,000-step pre-roll)
   for frames (observation='rgb') and symbolic vectors, in three patterns:
     plain      step() only;
     set_levels step(), then Env.set_levels on the envs that finished, drawn from 200 world seeds (the
                level-replay pattern: each new world is generated once, from the env's next episode on);
     reset      step(), then Env.reset(done, levels) with the same draws (the new level starts at once, so
                those envs' worlds are generated twice in that step);
     set_levels_abi  the set_levels pattern through cr_set_levels directly, without Env.set_levels' host-side
                checks: what the pattern costs on the device alone.
   Host wall clock over `--steps` steps ending in a device synchronise, so the host-side checks of set_levels
   (one device-to-host read of the chosen levels) are part of the number.  The patterns are timed
   alternately, `--reps` windows each, on envs of the same seed.

Prints the card's name and power limit, then one JSON line.

    python tools/levels_cost.py [--parent DIR] [--ab-reps 3] [--steps 500] [--reps 3]
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

PATTERNS = ('plain', 'set_levels', 'reset', 'set_levels_abi')


def card(index=0):
  return subprocess.run(['nvidia-smi', f'--id={index}', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                        capture_output=True, text=True, timeout=60).stdout.strip()


def bench_value(tree, steps, warmup):
  """bench.py's env-steps/s of the default workload, run from `tree`."""
  res = subprocess.run([sys.executable, 'bench.py', '--gpus', '1', '--steps', str(steps), '--warmup', str(warmup),
                        '--no-cpu-baseline'], cwd=str(tree), capture_output=True, text=True, timeout=1800)
  lines = [ln for ln in res.stdout.splitlines() if ln.startswith('{')]
  if res.returncode or not lines:
    raise RuntimeError(f'bench.py failed in {tree}: {res.stderr[-2000:]}')
  return json.loads(lines[-1])['value']


def ab(parent, reps, steps, warmup):
  out = {'parent': [], 'this': []}
  for _ in range(reps):
    out['parent'].append(bench_value(parent, steps, warmup))
    out['this'].append(bench_value(ROOT, steps, warmup))
  mean = {k: sum(v) / len(v) for k, v in out.items()}
  return {'env_steps_per_sec': {k: [round(x) for x in v] for k, v in out.items()},
          'spread': {k: round((max(v) - min(v)) / mean[k], 4) for k, v in out.items()},
          'this_over_parent': round(mean['this'] / mean['parent'], 4)}


def patterns(observation, args, device):
  import torch
  import crafter_b200
  kwargs = bench.env_kwargs(bench.CONFIGS['default'])
  B = kwargs['num_envs']
  T = 512
  gen = torch.Generator(device=device).manual_seed(1234)
  actions = torch.randint(0, 17, (T, B), generator=gen, device=device, dtype=torch.int32)
  pool = torch.randint(0, 2 ** 31 - 1, (200,), generator=gen, device=device, dtype=torch.int32)
  envs = {p: crafter_b200.Env(seed=0, auto_reset=True, device=device, observation=observation, **kwargs)
          for p in PATTERNS}
  draws = {p: torch.Generator(device=device).manual_seed(7) for p in PATTERNS}

  def one_step(env, p, t):
    done = env.step(actions[t % T])[2]
    if p == 'plain':
      return 0
    levels = pool[torch.randint(0, len(pool), (B,), generator=draws[p], device=device)]
    if p == 'set_levels':
      env.set_levels(levels, done)
    elif p == 'set_levels_abi':
      env._level_in.copy_(levels)
      env._level_mask.copy_(done)
      s = env._enter()
      env._lib.cr_set_levels(env._handle, env._level_mask.data_ptr(), env._level_in.data_ptr(), s)
      env._exit()
    else:
      env.reset(done, levels)
    return 1

  pos = args.preroll + args.warmup
  for p in PATTERNS:
    envs[p].reset()
    for t in range(pos):
      one_step(envs[p], p if t >= args.preroll else 'plain', t)  # the pre-roll itself is plain
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
  started = {p: int(envs[p].state['pstate'][:, bench_ps('episode')].sum()) for p in PATTERNS}
  for env in envs.values():
    env.close()
  mean = {p: sum(v) / len(v) for p, v in rates.items()}
  return {'env_steps_per_sec': {p: [round(x) for x in v] for p, v in rates.items()},
          'over_plain': {p: round(mean[p] / mean['plain'], 4) for p in PATTERNS}, 'episodes_started': started}


def bench_ps(name):
  from crafter_b200 import state as state_lib
  return state_lib.PS[name]


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--parent', help='a tree of the commit before levels, its library built (bench.py A/B)')
  ap.add_argument('--ab-reps', type=int, default=3)
  ap.add_argument('--bench-steps', type=int, default=2000)
  ap.add_argument('--bench-warmup', type=int, default=200)
  ap.add_argument('--steps', type=int, default=500)
  ap.add_argument('--warmup', type=int, default=50)
  ap.add_argument('--preroll', type=int, default=1000)
  ap.add_argument('--reps', type=int, default=3)
  args = ap.parse_args()
  gpu = card(0)
  print('card, power limit:', gpu, flush=True)
  out = {'gpu_and_power_limit': gpu}
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
