"""`-m gpu`: the workloads bench.py times, checked bit for bit against the C oracle at the batch size
they are timed at.

Every other bit-exact test runs at most 40 envs, where each grid-stride loop of the step (k_post's
balance CTAs, k_install, k_wg_mat, k_wg_obj, k_seed, k_terminal) runs a single round, and where
frame_partition never takes its aligned 16-byte branch (B >= 2048).  Here each entry of
bench.CONFIGS (and the default geometry at B = 4090 with terminal frames: a partial k_update CTA, a
partial last frame_partition thread) runs 1,300 auto-resetting steps from reset() with random
actions: the initial generation of every world, the synchronised start where every env balances on
steps 10, 20, ..., the first nightfall, and the desynchronised steady state bench.py measures after
its 1,000-step pre-roll.  Env i is the oracle's Env(seed=i).

Each step, for every env: done, reward, the player vector (inventory, achievements, vitals,
position, ...) and the step counter; the observation of a fixed sample of 512 envs (0 and B-1
included).  At checkpoints, for every env: observation, canonical state (oracle/canon.py) and
info['semantic'].  With final_obs: the terminal frame, semantic map, inventory, achievements,
position, length and death flag of every finished episode.  The default config runs steps 1001 to
1100 through Env.step_host with pinned buffers.  The output buffers are poisoned before every step,
so a frame the kernels never drew cannot pass as the previous step's copy.  The regime is asserted
(a step balancing more envs than num_sms * 4, nightfall, mixed night / day steps, regenerated
worlds), so that the test cannot pass without reaching it.

Runtime: 4.6 minutes for the file on an H100 SXM 80 GB (700 W limit) with 16 host threads for the
oracle (default 36 s, default at 4090 envs 39 s, view15 74 s, area256 118 s); most of it is the oracle
on the host.
"""
import time

import numpy as np
import pytest

import bench
from crafter_b200 import rules
from crafter_b200 import state as state_lib
from oracle import canon
from oracle import oracle_env
from tests.parity import POISON, frame_problem

pytestmark = pytest.mark.gpu

STEPS = 1300
SAMPLE = 512
HOST_STEPS = range(1001, 1101)  # step numbers run through Env.step_host (default config)
SEED = 0

CASES = {name: dict(bench.env_kwargs(cfg), final_obs=False) for name, cfg in bench.CONFIGS.items()}
CASES['default_b4090_final_obs'] = dict(bench.env_kwargs(bench.CONFIGS['default']), num_envs=4090, final_obs=True)

PS = state_lib.PS
# the 49 entries of the canonical player vector (oracle/canon.py)
PLAYER_FIELDS = list(rules.ITEMS) + list(rules.ACHIEVEMENTS) + [
    'hunger2', 'thirst2', 'fatigue', 'recover2', 'sleeping', 'facing', 'player_last_health', 'x', 'y',
    'env_last_health', 'unlocked']


def gpu_player(env):
  """The canonical player vectors of every env (state.canonical, vectorised) and the pstate rows."""
  st = env.state
  inv, ach = st['inventory'].cpu().numpy(), st['achievements'].cpu().numpy()
  ps = st['pstate'].cpu().numpy()
  facing = st['ents'][:, 1].contiguous().cpu().numpy().view(state_lib.ENT_DTYPE)['aux']
  cols = [ps[:, PS[k]] for k in ('hunger2', 'thirst2', 'fatigue', 'recover2', 'sleeping')] + [facing] + [
      ps[:, PS[k]] for k in ('player_last_health', 'player_x', 'player_y', 'env_last_health')] + [
      ps[:, PS['unlocked']].astype(np.int64) & 0xFFFFFFFF]
  vec = np.concatenate([inv.astype(np.int64), ach.astype(np.int64), np.stack(cols, 1).astype(np.int64)], 1)
  return vec, ps


def gpu_canonical(env, i, arrays):
  return state_lib.canonical(*(arrays[k][i] for k in ('mat', 'ents', 'inventory', 'achievements', 'pstate',
                                                       'touched')), env._area)


def check_rows(where, name, got, want, env_ids=None, fields=None):
  """Row i of `got` against row i of `want` (env env_ids[i]); names the first env and field that differ."""
  got, want = np.asarray(got), np.asarray(want)
  assert got.shape == want.shape, (where, name, got.shape, want.shape)
  bad = got != want
  if not bad.any():
    return
  row = int(np.argwhere(bad.reshape(len(bad), -1).any(1))[0][0])
  env = row if env_ids is None else int(env_ids[row])
  if got.ndim == 1:
    detail = f'{got[row]} vs oracle {want[row]}'
  else:
    cols = np.flatnonzero(bad[row].reshape(-1))[:8]
    names = [fields[c] if fields else int(c) for c in cols]
    detail = f'at {names}: {got[row].reshape(-1)[cols].tolist()} vs oracle {want[row].reshape(-1)[cols].tolist()}'
  raise AssertionError(f'{where} env {env} {name}: {detail} ({int(bad.reshape(len(bad), -1).any(1).sum())} envs differ)')


def check_frames(where, name, got, want, env_ids):
  for k, i in enumerate(env_ids):
    problem = frame_problem(got[k], want[k])
    assert problem is None, f'{where} env {int(i)} {name}: {problem}'


@pytest.mark.parametrize('case', sorted(CASES))
def test_full_batch_matches_oracle(case):
  import torch
  import crafter_b200
  kw = CASES[case]
  B, final_obs = kw['num_envs'], kw['final_obs']
  host_steps = HOST_STEPS if case == 'default' else ()
  geo = {k: kw[k] for k in ('area', 'view', 'size')}
  t0 = time.perf_counter()
  env = crafter_b200.Env(seed=SEED, auto_reset=True, **kw)
  oracle = oracle_env.OracleBatch(B, seed=SEED, **geo)
  dev = env.device
  num_sms = torch.cuda.get_device_properties(dev).multi_processor_count
  day = oracle_env.daylight_table(STEPS + 2)
  rs = np.random.RandomState(SEED)
  sample = np.sort(np.concatenate([[0, B - 1], 1 + np.random.RandomState(1).choice(B - 2, SAMPLE - 2, replace=False)]))
  sample_t = torch.as_tensor(sample, device=dev)
  h_a = torch.zeros(B, dtype=torch.int32).pin_memory()
  h_r = torch.zeros(B, dtype=torch.float32).pin_memory()
  h_d = torch.zeros(B, dtype=torch.bool).pin_memory()

  def poison():  # on the env's stream: the step (either entry point) is ordered behind it
    with torch.cuda.stream(env._stream):
      env._obs.fill_(POISON)
      if final_obs:
        env._final_obs.fill_(POISON)
        env._final_semantic.fill_(POISON)

  def checkpoint(where, obs):  # every env: state first (the most telling difference), then what is drawn from it
    arrays = {k: env.state[k].cpu().numpy() for k in ('mat', 'ents', 'inventory', 'achievements', 'pstate', 'touched')}
    for i in range(B):
      problem = canon.diff(oracle.envs[i].export_state(), gpu_canonical(env, i, arrays))
      assert problem is None, f'{where} env {i} state (oracle vs GPU): {problem}'
    check_rows(where, 'semantic', env.semantic().cpu().numpy(), oracle.semantic())
    check_frames(where, 'obs', obs.cpu().numpy(), oracle.render(), range(B))

  poison()
  obs = env.reset()
  oracle.reset(render=False)
  checkpoint(f'{case} reset', obs)
  age = np.zeros(B, np.int64)  # steps into the current episode (the oracle's env._step)
  checkpoints = {10, 20, 300, 1000, STEPS}
  first_night, max_balanced, night_frac, resets, terminal_frames = None, 0, [], 0, 0
  for n in range(1, STEPS + 1):
    where = f'{case} step {n}'
    actions = rs.randint(0, 17, B).astype(np.int32)
    poison()
    if n in host_steps:
      h_a.copy_(torch.from_numpy(actions))
      env.step_host(h_a, h_r, h_d)  # synchronises the env's stream
      obs, reward, done, info = env._obs, h_r.numpy().copy(), h_d.numpy().copy(), None
    else:
      obs, reward, done, info = env.step(torch.from_numpy(actions).to(dev))
      reward, done = reward.cpu().numpy(), done.cpu().numpy()
    _, ref_reward, ref_done = oracle.step(actions, auto_reset=False, render=False)
    age += 1
    check_rows(where, 'done', done, ref_done)
    check_rows(where, 'reward', reward, ref_reward.astype(np.float32))
    ended = np.flatnonzero(ref_done)
    ref_player = oracle.player()  # terminal rows for the envs that just ended
    if final_obs and len(ended):
      ended_t = torch.as_tensor(ended, device=dev)
      check_frames(where, 'final_observation', info['final_observation'][ended_t].cpu().numpy(),
                   oracle.render(ended), ended)
      check_rows(where, 'final_semantic', info['final_semantic'][ended_t].cpu().numpy(), oracle.semantic(ended), ended)
      check_rows(where, 'final_inventory', info['final_inventory'][ended_t].cpu().numpy(), ref_player[ended, :16], ended)
      check_rows(where, 'final_achievements', info['final_achievements'][ended_t].cpu().numpy(),
                 ref_player[ended, 16:38], ended)
      check_rows(where, 'final_player_pos', info['final_player_pos'][ended_t].cpu().numpy(),
                 ref_player[ended, 45:47], ended)
      fs = env.state['final_stats'][ended_t].cpu().numpy()
      check_rows(where, 'final length', fs[:, 22], age[ended], ended)
      check_rows(where, 'final death flag', fs[:, 23], (ref_player[ended, 0] <= 0).astype(np.int32), ended)
      terminal_frames += len(ended)
    if len(ended):
      oracle.reset(ended, render=False)
      ref_player[ended] = oracle.player(ended)
      age[ended] = 0
      resets += len(ended)
    got_player, ps = gpu_player(env)
    check_rows(where, 'player', got_player, ref_player, fields=PLAYER_FIELDS)
    check_rows(where, 'step counter', ps[:, PS['step']], age)
    # the regime this step ran in, from the device's step counters (checked equal to the oracle's above)
    max_balanced = max(max_balanced, int(((ps[:, PS['step']] > 0) & (ps[:, PS['step']] % 10 == 0)).sum()))
    nights = int((day[age] < 0.5).sum())
    night_frac.append(nights / B)
    if first_night is None and nights:
      first_night = n
      checkpoint(f'{where} (first night step)', obs)
    elif n in checkpoints:
      checkpoint(where, obs)
    else:
      check_frames(where, 'obs', obs[sample_t].cpu().numpy(), oracle.render(sample), sample)
  env.check_errors()
  night_frac = np.array(night_frac)
  print(f'{case}: B={B} {STEPS} steps in {time.perf_counter() - t0:.0f} s on {torch.cuda.get_device_name(dev)} '
        f'({oracle.threads} oracle threads): max balanced {max_balanced} (num_sms*4 = {4 * num_sms}), first night '
        f'step {first_night}, max night fraction {night_frac.max():.2f}, worlds regenerated {resets}, terminal '
        f'frames compared {terminal_frames}')
  assert max_balanced > 4 * num_sms, (case, 'no step balanced more envs than the balance CTAs', max_balanced)
  assert first_night is not None and night_frac.max() >= 0.5, (case, 'no night step', night_frac.max())
  assert ((night_frac >= 0.1) & (night_frac <= 0.9)).any(), (case, 'no mixed night / day step')
  assert resets >= (B if kw['area'][0] > 64 else 3 * B), (case, 'too few regenerated worlds', resets)
  if final_obs:
    assert terminal_frames >= B, (case, 'too few terminal frames compared', terminal_frames)
  env.close()
