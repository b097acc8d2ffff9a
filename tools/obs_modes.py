"""tools/obs_modes.py -- step time of Env(observation='rgb'), 'semantic' and 'symbolic' on one GPU, for each
workload of bench.CONFIGS, and of 'semantic' followed by the symbolic vector composed in torch from the state
tensors (what a user would write without the symbolic mode; `torch_symbolic` below).

bench.py's protocol: a 1,000-step pre-roll to the desynchronised steady state, a warm-up, then K steps, each
bracketed by CUDA events on the env's stream with the L2 flushed (256 MiB memset) between steps outside the
events.  The two modes are separate envs of the same seed and actions (so the same states), timed alternately
in the same process, `--reps` windows each; the torch composition is inside its step's events (the end event is
recorded on the stream the composition runs on).  Then the per-kernel times inside each step graph
(CRAFTER_B200_TIMING=2, bench.kernel_times) over the same steady-state snapshot; in the semantic graph the
`k_render` entry times k_local, in the symbolic graph k_symbolic, which replace the frame kernel there.  After the tick, the step has two
branches: the main one (k_post, then the frames or the windows) and world generation (k_install, k_wg_mat,
k_wg_obj); `main_ms` and `worldgen_ms` are their in-graph sums, measured while the branches share the SMs.

Prints the card's name and power limit, then one JSON line.

    python tools/obs_modes.py [--steps 500] [--warmup 50] [--reps 2] [--configs default area256 view15]
"""
import argparse
import json
import pathlib
import subprocess
import sys

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import bench  # noqa: E402

MODES = ('rgb', 'semantic', 'symbolic', 'semantic+torch')
DRAW = {'rgb': 'k_render', 'semantic': 'k_local', 'symbolic': 'k_symbolic'}  # the graph's `render` entry


def torch_symbolic(env):
  """The symbolic vector of every env composed with torch ops from the state tensors (gather of the window's
  materials and objects, one-hot, cast, concatenation): (B, D) float32, bit-equal to Env.symbolic()."""
  import torch
  import torch.nn.functional as F
  from crafter_b200.env import FACING, daylight_at
  st, (gx, gy), (w, h), dev = env.state, env._grid, env._area, env.device
  B, ps = env.num_envs, st['pstate']
  wx = ps[:, 12:13].long() + torch.arange(gx, device=dev) - gx // 2
  wy = ps[:, 13:14].long() + torch.arange(gy, device=dev) - gy // 2
  inside = (((wx >= 0) & (wx < w))[:, :, None] & ((wy >= 0) & (wy < h))[:, None, :]).reshape(B, -1, 1)
  cell = (wx.clamp(0, w - 1)[:, :, None] * h + wy.clamp(0, h - 1)[:, None, :]).reshape(B, -1)
  mat = st['mat'].gather(1, cell).long() & 0x7F
  slot = st['objmap'].gather(1, cell).long() & 0xFFFF
  ent = st['ents'].gather(1, slot)
  kind, aux = ent & 0xFF, ent >> 48
  ch = torch.where(kind == 5, 4 + aux, torch.where(kind == 6, torch.where(aux > 300, 9, 8), kind - 1))
  ch = torch.where(slot > 0, ch + 1, 0)
  cells = torch.cat([F.one_hot(mat, 13)[..., 1:], F.one_hot(ch, 11)[..., 1:]], -1) * inside
  return torch.cat([cells.reshape(B, -1).float(), st['inventory'].float() / 9,
                    F.one_hot(st['ents'][:, 1] >> 48, len(FACING)).float(), (ps[:, 4:5] != 0).float(),
                    daylight_at(ps, env._daylight)[:, None]], 1)


def card(index):
  return subprocess.run(['nvidia-smi', f'--id={index}', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                        capture_output=True, text=True, timeout=60).stdout.strip()


def timed_window(env, actions, start, steps, flush, compose=False):
  """Mean device ms per step over `steps` steps from action row `start` (bench.py's timed region); with
  `compose`, each step is followed by torch_symbolic inside the events."""
  import torch
  stream, dev = env._stream, env.device
  starts = [torch.cuda.Event(enable_timing=True) for _ in range(steps)]
  ends = [torch.cuda.Event(enable_timing=True) for _ in range(steps)]
  torch.cuda.synchronize(dev)
  for k in range(steps):
    env._actions.copy_(actions[(start + k) % len(actions)])
    flush.zero_()
    stream.wait_stream(torch.cuda.current_stream(dev))
    starts[k].record(stream)
    env.step(env.actions_buffer)
    if compose:
      torch_symbolic(env)
    ends[k].record(torch.cuda.current_stream(dev) if compose else stream)
  torch.cuda.synchronize(dev)
  return sum(s.elapsed_time(e) for s, e in zip(starts, ends)) / steps


def run_config(name, args, device):
  import torch
  import crafter_b200
  kwargs = bench.env_kwargs(bench.CONFIGS[name])
  B = kwargs['num_envs']
  T = 512
  gen = torch.Generator(device=device).manual_seed(1234)
  actions = torch.randint(0, 17, (T, B), generator=gen, device=device, dtype=torch.int32)
  flush = torch.empty(256 << 20, dtype=torch.uint8, device=device)
  envs = {m: crafter_b200.Env(seed=0, auto_reset=True, device=device, observation=m.split('+')[0], **kwargs)
          for m in MODES}
  pos = args.preroll + args.warmup
  for m, env in envs.items():
    env.reset()
    for t in range(pos):
      env.step(actions[t % T])
      if m.endswith('+torch') and t >= args.preroll:  # the warm-up covers the composition's kernels too
        torch_symbolic(env)
  torch.cuda.synchronize(device)
  ms = {m: [] for m in MODES}
  for _ in range(args.reps):
    for m in MODES:  # alternately, the same action rows for all
      ms[m].append(timed_window(envs[m], actions, pos, args.steps, flush, compose=m.endswith('+torch')))
    pos += args.steps
  same = all(bool((envs['rgb'].state[k] == envs[m].state[k]).all()) for m in MODES for k in ('mat', 'pstate', 'ents'))
  torch_matches = bool((torch_symbolic(envs['symbolic']).view(torch.int32) == envs['symbolic'].symbolic().view(torch.int32)).all())
  snapshot = envs['semantic'].state_dict()
  kernels = {}
  for m in DRAW:
    n, times = bench.kernel_times(dict(kwargs, observation=m), 0, 0, snapshot, actions[pos % T:], args.kernel_steps)
    if 'k_render' in times:
      times[DRAW[m]] = times.pop('k_render')
    draw = times.get(DRAW[m], 0.0)
    kernels[m] = dict(steps=n, ms=times, main_ms=times.get('k_post', 0.0) + draw,
                      worldgen_ms=sum(times.get(k, 0.0) for k in ('k_install', 'k_wg_mat', 'k_wg_obj')))
  for env in envs.values():
    env.close()
  mean = {m: sum(v) / len(v) for m, v in ms.items()}
  return {
      'num_envs': B, 'area': kwargs['area'], 'view': kwargs['view'], 'size': kwargs['size'],
      'ms_per_step': {m: [round(v, 4) for v in ms[m]] for m in MODES},
      'env_steps_per_sec': {m: round(B / (mean[m] * 1e-3)) for m in MODES},
      'semantic_speedup': round(mean['rgb'] / mean['semantic'], 3),
      'symbolic_speedup': round(mean['rgb'] / mean['symbolic'], 3),
      'torch_composition_over_symbolic': round(mean['semantic+torch'] / mean['symbolic'], 3),
      'same_states': same, 'torch_composition_bit_equal': torch_matches, 'in_graph': kernels}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=500)
  ap.add_argument('--warmup', type=int, default=50)
  ap.add_argument('--preroll', type=int, default=1000)
  ap.add_argument('--reps', type=int, default=2)
  ap.add_argument('--kernel-steps', type=int, default=100)
  ap.add_argument('--configs', nargs='*', default=list(bench.CONFIGS), choices=list(bench.CONFIGS))
  args = ap.parse_args()
  import torch
  device = torch.device('cuda', 0)
  torch.cuda.set_device(device)
  gpu = card(0)
  print('card, power limit:', gpu, flush=True)
  out = {'gpu_and_power_limit': gpu, 'steps': args.steps, 'warmup': args.warmup, 'preroll': args.preroll,
         'reps': args.reps, 'l2': 'flushed between timed steps (256 MiB memset outside the per-step CUDA events)',
         'configs': {}}
  for name in args.configs:
    out['configs'][name] = run_config(name, args, device)
    print(name, json.dumps(out['configs'][name]), flush=True)
  print(json.dumps(out))


if __name__ == '__main__':
  main()
