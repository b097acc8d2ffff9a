"""`-m gpu`: observation='semantic' on the H100 against the C oracle, at the batch sizes bench.py times and across
the geometry sweep.

test_full_batch_semantic_matches_oracle runs each workload of bench.CONFIGS (and the default geometry at
B = 4090 with terminal windows) for 1,300 auto-resetting random-policy steps from reset(), as
tests/test_full_batch_gpu.py does with frames.  Every step, for every env: the window, done, reward, the player
vector, the step counter and the info entries 'facing', 'sleeping' and 'daylight'; every terminal window and
terminal semantic map.  The output buffers are poisoned before every step.  At the checkpoints of
test_full_batch_gpu.py, for every env: the canonical state and render() frames (drawn from the state alone,
without the views k_view prepares inside a frame step, which a semantic step does not run).  The same regime
is asserted.

test_semantic_geometry_sweep_matches_oracle runs each geometry of tests/test_semantic_obs.py at
B = 8 * num_sms + 1 across nightfall, with the start states of tests/test_geometry_sweep_gpu.py: windows,
terminal windows (at every geometry, those where terminal frames are rejected included), done, reward, player
vector and step counter every step; canonical state and info['semantic'] at three checkpoints.

Runtime: 5.2 to 5.7 minutes for the file on an H100 80 GB HBM3 at a 400 W limit (in the faster run: area256
126 s, view15 49 s, default at 4090 envs 43 s, default 38 s, the sweep 48 s); most of it is the oracle on the
host.
"""
import time

import numpy as np
import pytest

import bench
from crafter_b200 import state as state_lib
from crafter_b200.env import FACING
from oracle import canon
from oracle import oracle_env
from tests.test_full_batch_gpu import PLAYER_FIELDS, POISON, check_frames, check_rows, gpu_canonical, gpu_player
from tests.test_geometry_sweep_gpu import start_state
from tests.test_schedule_knobs import SLEEP, SLEEPING
from tests.test_semantic_obs import CASES as SWEEP, FACING_IDX, PX, PY, expected_windows, grid_of

pytestmark = pytest.mark.gpu

STEPS = 1300
SEED = 0
CASES = {name: dict(bench.env_kwargs(cfg), final_obs=False) for name, cfg in bench.CONFIGS.items()}
CASES['default_b4090_final_obs'] = dict(bench.env_kwargs(bench.CONFIGS['default']), num_envs=4090, final_obs=True)
FACING_TABLE = np.array(FACING, np.int32)
PS = state_lib.PS


def oracle_windows(oracle, player, grid, ids=None):
  """The windows of the oracle envs `ids` (all when None) from their info['semantic'] and player vectors."""
  return expected_windows(oracle.semantic(ids), player[:, PX], player[:, PY], grid)


def check_info(where, info, player, steps, day):
  """info['facing'] / ['sleeping'] / ['daylight'] against the oracle's player vectors and daylight table."""
  check_rows(where, 'facing', info['facing'].cpu().numpy(), FACING_TABLE[player[:, FACING_IDX]])
  check_rows(where, 'sleeping', info['sleeping'].cpu().numpy(), player[:, SLEEPING] != 0)
  check_rows(where, 'daylight', info['daylight'].cpu().numpy(), day[steps].astype(np.float32))


def make_poison(env, final_obs):
  import torch

  def poison():  # on the env's stream: the step is ordered behind it
    with torch.cuda.stream(env._stream):
      env._local.fill_(POISON)
      if final_obs:
        env._final_local.fill_(POISON)
        env._final_semantic.fill_(POISON)
  return poison


@pytest.mark.parametrize('case', sorted(CASES))
def test_full_batch_semantic_matches_oracle(case):
  import torch
  import crafter_b200
  kw = CASES[case]
  B, final_obs = kw['num_envs'], kw['final_obs']
  geo = {k: kw[k] for k in ('area', 'view', 'size')}
  grid = grid_of(geo['view'])
  t0 = time.perf_counter()
  env = crafter_b200.Env(seed=SEED, auto_reset=True, observation='semantic', **kw)
  assert env.observation_space == crafter_b200.env.BoxSpace(0, 18, grid, np.uint8)
  oracle = oracle_env.OracleBatch(B, seed=SEED, **geo)
  dev = env.device
  num_sms = torch.cuda.get_device_properties(dev).multi_processor_count
  day = oracle_env.daylight_table(STEPS + 2)
  rs = np.random.RandomState(SEED)
  poison = make_poison(env, final_obs)

  def checkpoint(where):  # every env: state, then the frames render() draws from it alone
    arrays = {k: env.state[k].cpu().numpy() for k in ('mat', 'ents', 'inventory', 'achievements', 'pstate', 'touched')}
    for i in range(B):
      problem = canon.diff(oracle.envs[i].export_state(), gpu_canonical(env, i, arrays))
      assert problem is None, f'{where} env {i} state (oracle vs GPU): {problem}'
    check_frames(where, 'render()', env.render().cpu().numpy(), oracle.render(), range(B))

  poison()
  local = env.reset()
  oracle.reset(render=False)
  check_rows(f'{case} reset', 'window', local.cpu().numpy(), oracle_windows(oracle, oracle.player(), grid))
  checkpoint(f'{case} reset')
  age = np.zeros(B, np.int64)
  checkpoints = {10, 20, 300, 1000, STEPS}
  first_night, max_balanced, night_frac, resets, terminal_windows = None, 0, [], 0, 0
  for n in range(1, STEPS + 1):
    where = f'{case} step {n}'
    actions = rs.randint(0, 17, B).astype(np.int32)
    poison()
    local, reward, done, info = env.step(torch.from_numpy(actions).to(dev))
    local, reward, done = local.cpu().numpy(), reward.cpu().numpy(), done.cpu().numpy()
    _, ref_reward, ref_done = oracle.step(actions, auto_reset=False, render=False)
    age += 1
    check_rows(where, 'done', done, ref_done)
    check_rows(where, 'reward', reward, ref_reward.astype(np.float32))
    ended = np.flatnonzero(ref_done)
    ref_player = oracle.player()
    if final_obs and len(ended):
      ended_t = torch.as_tensor(ended, device=dev)
      check_rows(where, 'final_observation (terminal window)', info['final_observation'][ended_t].cpu().numpy(),
                 oracle_windows(oracle, ref_player[ended], grid, ended), ended)
      check_rows(where, 'final_semantic', info['final_semantic'][ended_t].cpu().numpy(), oracle.semantic(ended), ended)
      terminal_windows += len(ended)
    if len(ended):
      oracle.reset(ended, render=False)
      ref_player[ended] = oracle.player(ended)
      age[ended] = 0
      resets += len(ended)
    got_player, ps = gpu_player(env)
    check_rows(where, 'player', got_player, ref_player, fields=PLAYER_FIELDS)
    check_rows(where, 'step counter', ps[:, PS['step']], age)
    check_info(where, info, ref_player, age, day)  # lazy: the state the step returned, regenerated envs included
    check_rows(where, 'window', local, oracle_windows(oracle, ref_player, grid))
    max_balanced = max(max_balanced, int(((age > 0) & (age % 10 == 0)).sum()))
    nights = int((day[age] < 0.5).sum())
    night_frac.append(nights / B)
    if first_night is None and nights:
      first_night = n
      checkpoint(f'{where} (first night step)')
    elif n in checkpoints:
      checkpoint(where)
  env.check_errors()
  night_frac = np.array(night_frac)
  print(f'{case}: B={B} {STEPS} semantic steps in {time.perf_counter() - t0:.0f} s on '
        f'{torch.cuda.get_device_name(dev)} ({oracle.threads} oracle threads): max balanced {max_balanced} '
        f'(num_sms*4 = {4 * num_sms}), first night step {first_night}, max night fraction {night_frac.max():.2f}, '
        f'worlds regenerated {resets}, terminal windows compared {terminal_windows}')
  assert max_balanced > 4 * num_sms, (case, 'no step balanced more envs than the balance CTAs', max_balanced)
  assert first_night is not None and night_frac.max() >= 0.5, (case, 'no night step', night_frac.max())
  assert ((night_frac >= 0.1) & (night_frac <= 0.9)).any(), (case, 'no mixed night / day step')
  assert resets >= (B if kw['area'][0] > 64 else 3 * B), (case, 'too few regenerated worlds', resets)
  if final_obs:
    assert terminal_windows >= B, (case, 'too few terminal windows compared', terminal_windows)
  env.close()


SWEEP_LENGTH, SWEEP_STEPS = 160, 45


@pytest.mark.parametrize('name', list(SWEEP))
def test_semantic_geometry_sweep_matches_oracle(name):
  import torch
  import crafter_b200
  geo = SWEEP[name]
  grid = grid_of(geo['view'])
  num_sms = torch.cuda.get_device_properties(0).multi_processor_count
  B = 8 * num_sms + 1
  t0 = time.perf_counter()
  env = crafter_b200.Env(num_envs=B, seed=0, length=SWEEP_LENGTH, auto_reset=True, final_obs=True,
                         observation='semantic', **geo)
  oracle = oracle_env.OracleBatch(B, seed=0, length=SWEEP_LENGTH, **geo)
  dev = env.device
  day = oracle_env.daylight_table(SWEEP_LENGTH + 2)
  poison = make_poison(env, True)

  def checkpoint(where):
    arrays = {k: env.state[k].cpu().numpy() for k in ('mat', 'ents', 'inventory', 'achievements', 'pstate', 'touched')}
    for i in range(B):
      problem = canon.diff(oracle.envs[i].export_state(), gpu_canonical(env, i, arrays))
      assert problem is None, f'{where} env {i} state (oracle vs GPU): {problem}'
    check_rows(where, 'semantic', env.semantic().cpu().numpy(), oracle.semantic())

  poison()
  local = env.reset()
  oracle.reset(render=False)
  check_rows(f'{name} reset', 'window', local.cpu().numpy(), oracle_windows(oracle, oracle.player(), grid))
  age = start_state(env, oracle, 0, B)
  rs = np.random.RandomState(7)
  max_balanced, night_frac, resets, terminal_windows, sleeping_night = 0, [], 0, 0, 0
  for n in range(1, SWEEP_STEPS + 1):
    where = f'{name} step {n}'
    actions = rs.randint(0, 17, B).astype(np.int32)
    actions[rs.rand(B) < 0.3] = SLEEP
    poison()
    local, reward, done, info = env.step(torch.from_numpy(actions).to(dev))
    local, reward, done = local.cpu().numpy(), reward.cpu().numpy(), done.cpu().numpy()
    _, ref_reward, ref_done = oracle.step(actions, auto_reset=False, render=False)
    age += 1
    check_rows(where, 'done', done, ref_done)
    check_rows(where, 'reward', reward, ref_reward.astype(np.float32))
    ended = np.flatnonzero(ref_done)
    ref_player = oracle.player()
    if len(ended):
      ended_t = torch.as_tensor(ended, device=dev)
      check_rows(where, 'final_observation (terminal window)', info['final_observation'][ended_t].cpu().numpy(),
                 oracle_windows(oracle, ref_player[ended], grid, ended), ended)
      check_rows(where, 'final_semantic', info['final_semantic'][ended_t].cpu().numpy(), oracle.semantic(ended), ended)
      terminal_windows += len(ended)
      oracle.reset(ended, render=False)
      ref_player[ended] = oracle.player(ended)
      age[ended] = 0
      resets += len(ended)
    got_player, ps = gpu_player(env)
    check_rows(where, 'player', got_player, ref_player, fields=PLAYER_FIELDS)
    check_rows(where, 'step counter', ps[:, PS['step']], age)
    check_info(where, info, ref_player, age, day)  # lazy: the state the step returned, regenerated envs included
    check_rows(where, 'window', local, oracle_windows(oracle, ref_player, grid))
    max_balanced = max(max_balanced, int(((age > 0) & (age % 10 == 0)).sum()))
    night = day[age] < 0.5
    night_frac.append(night.mean())
    sleeping_night += int((night & (ref_player[:, SLEEPING] != 0)).sum())
    if n in (1, 25, SWEEP_STEPS):
      checkpoint(where)
  env.check_errors()
  night_frac = np.array(night_frac)
  print(f'{name}: B={B} {SWEEP_STEPS} semantic steps in {time.perf_counter() - t0:.0f} s: max balanced {max_balanced}, '
        f'night fraction {night_frac.min():.2f}..{night_frac.max():.2f}, sleeping night steps {sleeping_night}, '
        f'worlds regenerated {resets}, terminal windows compared {terminal_windows}')
  assert max_balanced > 4 * num_sms, (name, 'no step balanced more envs than the balance CTAs', max_balanced)
  assert ((night_frac >= 0.1) & (night_frac <= 0.9)).any(), (name, 'no mixed night / day step')
  assert sleeping_night > 0, (name, 'no night step of a sleeping player')
  assert resets >= B and terminal_windows >= B, (name, 'too few terminal windows compared', resets, terminal_windows)
  env.close()


def test_one_handle_serves_both_kinds_of_step():
  """Frame steps and window steps alternate on one handle (cr_step, cr_step_local), each against the oracle;
  Env.local_semantic() and info['local_semantic'] in 'rgb' mode; step_host refused in 'semantic' mode."""
  import torch
  import crafter_b200
  from crafter_b200 import _cabi
  B, length, grid = 64, 12, grid_of((9, 9))
  env = crafter_b200.Env(num_envs=B, seed=3, length=length, auto_reset=True, final_obs=True)
  oracle = oracle_env.OracleBatch(B, seed=3, length=length)
  local = torch.empty(B, *grid, dtype=torch.uint8, device=env.device)
  env.reset()
  oracle.reset(render=False)
  rs = np.random.RandomState(4)
  for n in range(40):
    actions = rs.randint(0, 17, B).astype(np.int32)
    env.actions_buffer.copy_(torch.from_numpy(actions))
    if n % 2:
      local.fill_(POISON)
      s = env._enter()
      _cabi.check(env._lib.cr_step_local(env._handle, env._ptrs[0], local.data_ptr(), env._ptrs[2], env._ptrs[3], s))
      env._exit()
      done = env._done.cpu().numpy()
    else:
      obs, _, done, info = env.step(env.actions_buffer)
      done = done.cpu().numpy()
    _, _, ref_done = oracle.step(actions, auto_reset=False, render=False)
    check_rows(f'step {n}', 'done', done, ref_done)
    ended = np.flatnonzero(ref_done)
    if len(ended):
      oracle.reset(ended, render=False)
    player = oracle.player()
    want = oracle_windows(oracle, player, grid)
    if n % 2:
      check_rows(f'step {n}', 'window (cr_step_local)', local.cpu().numpy(), want)
    else:
      check_frames(f'step {n}', 'obs', obs.cpu().numpy(), oracle.render(), range(B))
      check_rows(f'step {n}', "info['local_semantic']", info['local_semantic'].cpu().numpy(), want)
    check_rows(f'step {n}', 'local_semantic()', env.local_semantic().cpu().numpy(), want)
  env.close()
  sem = crafter_b200.Env(num_envs=4, seed=1, observation='semantic')
  sem.reset()
  pinned = [torch.zeros(4, dtype=d).pin_memory() for d in (torch.int32, torch.float32, torch.bool)]
  with pytest.raises(RuntimeError, match='not available'):
    sem.step_host(*pinned)
  with pytest.raises(ValueError, match='image'):
    crafter_b200.recorder.EpisodeRecorder(sem, '/nonexistent-not-created')
  sem.close()


def test_vector_env_semantic_spaces_and_final_obs():
  import torch
  from crafter_b200 import vector
  B, length, grid = 8, 3, grid_of((9, 9))
  venv = vector.make('CrafterReward-v1', num_envs=B, seed=0, length=length, observation='semantic')
  assert tuple(venv.single_observation_space.shape) == grid and tuple(venv.observation_space.shape) == (B,) + grid
  assert int(np.max(venv.single_observation_space.high)) == 18
  oracle = oracle_env.OracleBatch(B, seed=0, length=length)
  obs, _ = venv.reset()
  oracle.reset(render=False)
  check_rows('vector reset', 'window', obs.cpu().numpy(), oracle_windows(oracle, oracle.player(), grid))
  finals = 0
  for n in range(2 * length):
    actions = np.full(B, 0, np.int32)
    obs, reward, terminated, truncated, info = venv.step(torch.from_numpy(actions).to(venv.env.device))
    _, _, ref_done = oracle.step(actions, auto_reset=False, render=False)
    ended = np.flatnonzero(ref_done)
    if len(ended):
      player = oracle.player(ended)
      check_rows(f'vector step {n}', 'final_obs', info['final_obs'].cpu().numpy()[ended],
                 oracle_windows(oracle, player, grid, ended), ended)
      assert info['_final_obs'].cpu().numpy()[ended].all()
      finals += len(ended)
      oracle.reset(ended, render=False)
    check_rows(f'vector step {n}', 'window', obs.cpu().numpy(), oracle_windows(oracle, oracle.player(), grid))
  assert finals == 2 * B
  venv.close()
