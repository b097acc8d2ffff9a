"""`-m gpu`: observation='symbolic' on the H100 against the C oracle, at the batch sizes bench.py times and across
the geometry sweep.  The expected vector is the restatement of tests/test_symbolic_obs.py (expected_vector) from
the oracle's canonical state and daylight; vectors are compared bit for bit.

test_full_batch_symbolic_matches_oracle runs each workload of bench.CONFIGS (and the default geometry at
B = 4090 with terminal vectors) for 1,300 auto-resetting random-policy steps from reset().  Every step, for
every env: done and reward; the vector of a fixed sample of 512 envs (0 and B - 1 included); every terminal
vector and terminal semantic map.  At the checkpoints of tests/test_full_batch_gpu.py, for every env: the
vector and the canonical state.  The output buffers are filled with 0xFF bytes (NaN) before every step, so an
entry the kernels never wrote cannot pass.  The regime (balance beyond the balance CTAs, nightfall, mixed steps,
regenerated worlds) is asserted.

test_symbolic_geometry_sweep_matches_oracle runs each geometry of tests/test_semantic_obs.py at
B = 8 * num_sms + 1 across nightfall: vectors and terminal vectors of every env every step.

Runtime: about 11.5 minutes for the file on an H100 80 GB HBM3 with 16 host threads for the oracle, measured
in two runs (area256 201 s, default 102 s, default at 4090 envs 101 s at a 400 W limit; view15 153 s, the sweep
118 s, the rest 7 s at a 700 W limit); most of it is the oracle and the numpy restatement on the host.
"""
import time

import numpy as np
import pytest

import bench
from crafter_b200.env import symbolic_layout
from oracle import canon
from oracle import oracle_env
from tests.test_full_batch_gpu import POISON, check_frames, check_rows, gpu_canonical
from tests.test_geometry_sweep_gpu import start_state
from tests.test_schedule_knobs import SLEEP
from tests.test_semantic_obs import CASES as SWEEP, grid_of
from tests.test_semantic_obs_gpu import oracle_windows
from tests.test_symbolic_obs import expected_vector, vector_problem

pytestmark = pytest.mark.gpu

STEPS = 1300
SAMPLE = 512
SEED = 0
NAN_BYTES = 0xFF  # vector buffers are filled with it before a step: a float32 of 0xFF bytes is a NaN, equal to nothing
CASES = {name: dict(bench.env_kwargs(cfg), final_obs=False) for name, cfg in bench.CONFIGS.items()}
CASES['default_b4090_final_obs'] = dict(bench.env_kwargs(bench.CONFIGS['default']), num_envs=4090, final_obs=True)


def oracle_vectors(oracle, grid, ids):
  """The restated vectors of the oracle envs `ids`: (len(ids), D) float32."""
  out = []
  for i in ids:
    st = oracle.envs[int(i)].export_state()
    out.append(expected_vector(st, st['daylight'], grid))
  return np.stack(out)


def check_vectors(where, name, got, want, ids, grid):
  """Bit for bit; names the first env, part and channel that differ."""
  for k, i in enumerate(ids):
    problem = vector_problem(got[k], want[k], grid)
    assert problem is None, f'{where} env {int(i)} {name}: {problem}'


def make_poison(env, final_obs):
  import torch

  def poison():  # on the env's stream: the step is ordered behind it
    with torch.cuda.stream(env._stream):
      env._sym.view(torch.uint8).fill_(NAN_BYTES)
      if final_obs:
        env._final_symbolic.view(torch.uint8).fill_(NAN_BYTES)
        env._final_semantic.fill_(POISON)
  return poison


@pytest.mark.parametrize('case', sorted(CASES))
def test_full_batch_symbolic_matches_oracle(case):
  import torch
  import crafter_b200
  kw = CASES[case]
  B, final_obs = kw['num_envs'], kw['final_obs']
  geo = {k: kw[k] for k in ('area', 'view', 'size')}
  grid = grid_of(geo['view'])
  dim = symbolic_layout(grid)['daylight'].stop
  t0 = time.perf_counter()
  env = crafter_b200.Env(seed=SEED, auto_reset=True, observation='symbolic', **kw)
  assert env.observation_space == crafter_b200.env.BoxSpace(0, 1, (dim,), np.float32)
  oracle = oracle_env.OracleBatch(B, seed=SEED, **geo)
  dev = env.device
  num_sms = torch.cuda.get_device_properties(dev).multi_processor_count
  day = oracle_env.daylight_table(STEPS + 2)
  rs = np.random.RandomState(SEED)
  sample = np.sort(np.concatenate([[0, B - 1], 1 + np.random.RandomState(1).choice(B - 2, SAMPLE - 2, replace=False)]))
  everyone = np.arange(B)
  poison = make_poison(env, final_obs)

  def checkpoint(where, vec):  # every env: vector and state
    check_vectors(where, 'vector', vec, oracle_vectors(oracle, grid, everyone), everyone, grid)
    arrays = {k: env.state[k].cpu().numpy() for k in ('mat', 'ents', 'inventory', 'achievements', 'pstate', 'touched')}
    for i in range(B):
      problem = canon.diff(oracle.envs[i].export_state(), gpu_canonical(env, i, arrays))
      assert problem is None, f'{where} env {i} state (oracle vs GPU): {problem}'

  poison()
  vec = env.reset()
  oracle.reset(render=False)
  checkpoint(f'{case} reset', vec.cpu().numpy())
  age = np.zeros(B, np.int64)
  checkpoints = {10, 20, 300, 1000, STEPS}
  first_night, max_balanced, night_frac, resets, terminal_vectors = None, 0, [], 0, 0
  for n in range(1, STEPS + 1):
    where = f'{case} step {n}'
    actions = rs.randint(0, 17, B).astype(np.int32)
    poison()
    vec, reward, done, info = env.step(torch.from_numpy(actions).to(dev))
    vec, reward, done = vec.cpu().numpy(), reward.cpu().numpy(), done.cpu().numpy()
    _, ref_reward, ref_done = oracle.step(actions, auto_reset=False, render=False)
    age += 1
    check_rows(where, 'done', done, ref_done)
    check_rows(where, 'reward', reward, ref_reward.astype(np.float32))
    ended = np.flatnonzero(ref_done)
    if final_obs and len(ended):
      ended_t = torch.as_tensor(ended, device=dev)
      check_vectors(where, 'final_observation (terminal vector)', info['final_observation'][ended_t].cpu().numpy(),
                    oracle_vectors(oracle, grid, ended), ended, grid)
      check_rows(where, 'final_semantic', info['final_semantic'][ended_t].cpu().numpy(), oracle.semantic(ended), ended)
      terminal_vectors += len(ended)
    if len(ended):
      oracle.reset(ended, render=False)
      age[ended] = 0
      resets += len(ended)
    nights = int((day[age] < 0.5).sum())
    night_frac.append(nights / B)
    max_balanced = max(max_balanced, int(((age > 0) & (age % 10 == 0)).sum()))
    if first_night is None and nights:
      first_night = n
      checkpoint(f'{where} (first night step)', vec)
    elif n in checkpoints:
      checkpoint(where, vec)
    else:
      check_vectors(where, 'vector', vec[sample], oracle_vectors(oracle, grid, sample), sample, grid)
  env.check_errors()
  night_frac = np.array(night_frac)
  print(f'{case}: B={B} D={dim} {STEPS} symbolic steps in {time.perf_counter() - t0:.0f} s on '
        f'{torch.cuda.get_device_name(dev)} ({oracle.threads} oracle threads): max balanced {max_balanced}, '
        f'first night step {first_night}, max night fraction {night_frac.max():.2f}, worlds regenerated {resets}, '
        f'terminal vectors compared {terminal_vectors}')
  assert max_balanced > 4 * num_sms, (case, 'no step balanced more envs than the balance CTAs', max_balanced)
  assert first_night is not None and night_frac.max() >= 0.5, (case, 'no night step', night_frac.max())
  assert ((night_frac >= 0.1) & (night_frac <= 0.9)).any(), (case, 'no mixed night / day step')
  assert resets >= (B if kw['area'][0] > 64 else 3 * B), (case, 'too few regenerated worlds', resets)
  if final_obs:
    assert terminal_vectors >= B, (case, 'too few terminal vectors compared', terminal_vectors)
  env.close()


SWEEP_LENGTH, SWEEP_STEPS = 160, 45


@pytest.mark.parametrize('name', list(SWEEP))
def test_symbolic_geometry_sweep_matches_oracle(name):
  import torch
  import crafter_b200
  geo = SWEEP[name]
  grid = grid_of(geo['view'])
  num_sms = torch.cuda.get_device_properties(0).multi_processor_count
  B = 8 * num_sms + 1
  everyone = np.arange(B)
  t0 = time.perf_counter()
  env = crafter_b200.Env(num_envs=B, seed=0, length=SWEEP_LENGTH, auto_reset=True, final_obs=True,
                         observation='symbolic', **geo)
  oracle = oracle_env.OracleBatch(B, seed=0, length=SWEEP_LENGTH, **geo)
  dev = env.device
  day = oracle_env.daylight_table(SWEEP_LENGTH + 2)
  poison = make_poison(env, True)
  poison()
  vec = env.reset()
  oracle.reset(render=False)
  check_vectors(f'{name} reset', 'vector', vec.cpu().numpy(), oracle_vectors(oracle, grid, everyone), everyone, grid)
  age = start_state(env, oracle, 0, B)
  rs = np.random.RandomState(7)
  night_frac, resets, terminal_vectors = [], 0, 0
  for n in range(1, SWEEP_STEPS + 1):
    where = f'{name} step {n}'
    actions = rs.randint(0, 17, B).astype(np.int32)
    actions[rs.rand(B) < 0.3] = SLEEP
    poison()
    vec, reward, done, info = env.step(torch.from_numpy(actions).to(dev))
    vec, reward, done = vec.cpu().numpy(), reward.cpu().numpy(), done.cpu().numpy()
    _, ref_reward, ref_done = oracle.step(actions, auto_reset=False, render=False)
    age += 1
    check_rows(where, 'done', done, ref_done)
    check_rows(where, 'reward', reward, ref_reward.astype(np.float32))
    ended = np.flatnonzero(ref_done)
    if len(ended):
      ended_t = torch.as_tensor(ended, device=dev)
      check_vectors(where, 'final_observation (terminal vector)', info['final_observation'][ended_t].cpu().numpy(),
                    oracle_vectors(oracle, grid, ended), ended, grid)
      check_rows(where, 'final_semantic', info['final_semantic'][ended_t].cpu().numpy(), oracle.semantic(ended), ended)
      terminal_vectors += len(ended)
      oracle.reset(ended, render=False)
      age[ended] = 0
      resets += len(ended)
    check_vectors(where, 'vector', vec, oracle_vectors(oracle, grid, everyone), everyone, grid)
    night_frac.append((day[age] < 0.5).mean())
  env.check_errors()
  night_frac = np.array(night_frac)
  print(f'{name}: B={B} {SWEEP_STEPS} symbolic steps in {time.perf_counter() - t0:.0f} s: night fraction '
        f'{night_frac.min():.2f}..{night_frac.max():.2f}, worlds regenerated {resets}, terminal vectors compared '
        f'{terminal_vectors}')
  assert ((night_frac >= 0.1) & (night_frac <= 0.9)).any(), (name, 'no mixed night / day step')
  assert resets >= B and terminal_vectors >= B, (name, 'too few terminal vectors compared', resets, terminal_vectors)
  env.close()


def test_one_handle_serves_three_kinds_of_step():
  """Frame, window and vector steps rotate on one handle (cr_step, cr_step_local, cr_step_symbolic; terminal
  frames on), each against the oracle, and the vector steps also against an env of the same seed that takes
  only vector steps; Env.symbolic() in 'rgb' mode; step_host refused in 'symbolic' mode."""
  import torch
  import crafter_b200
  from crafter_b200 import _cabi
  B, length, grid = 64, 12, grid_of((9, 9))
  dim = symbolic_layout(grid)['daylight'].stop
  everyone = np.arange(B)
  env = crafter_b200.Env(num_envs=B, seed=3, length=length, auto_reset=True, final_obs=True)
  only = crafter_b200.Env(num_envs=B, seed=3, length=length, auto_reset=True, observation='symbolic')
  oracle = oracle_env.OracleBatch(B, seed=3, length=length)
  local = torch.empty(B, *grid, dtype=torch.uint8, device=env.device)
  vec = torch.empty(B, dim, dtype=torch.float32, device=env.device)
  env.reset()
  only.reset()
  oracle.reset(render=False)
  rs = np.random.RandomState(4)
  launches = []
  for n in range(45):
    actions = rs.randint(0, 17, B).astype(np.int32)
    env.actions_buffer.copy_(torch.from_numpy(actions))
    before = env.launch_count
    kind = n % 3
    if kind == 0:
      obs, _, done, info = env.step(env.actions_buffer)
    else:
      out, fn = (local, env._lib.cr_step_local) if kind == 1 else (vec, env._lib.cr_step_symbolic)
      out.view(torch.uint8).fill_(NAN_BYTES if kind == 2 else POISON)
      s = env._enter()
      _cabi.check(fn(env._handle, env._ptrs[0], out.data_ptr(), env._ptrs[2], env._ptrs[3], s))
      env._exit()
      done = env._done
    launches.append((kind, env.launch_count - before))
    done = done.cpu().numpy()
    only_vec = only.step(torch.from_numpy(actions).to(only.device))[0].cpu().numpy()
    _, _, ref_done = oracle.step(actions, auto_reset=False, render=False)
    check_rows(f'step {n}', 'done', done, ref_done)
    ended = np.flatnonzero(ref_done)
    if len(ended):
      oracle.reset(ended, render=False)
    want = oracle_vectors(oracle, grid, everyone)
    check_vectors(f'step {n}', 'vector (symbolic-only env)', only_vec, want, everyone, grid)
    if kind == 0:
      check_frames(f'step {n}', 'obs', obs.cpu().numpy(), oracle.render(), range(B))
      check_vectors(f'step {n}', 'Env.symbolic()', env.symbolic().cpu().numpy(), want, everyone, grid)
    elif kind == 1:
      check_rows(f'step {n}', 'window (cr_step_local)', local.cpu().numpy(), oracle_windows(oracle, oracle.player(), grid))
    else:
      check_rows(f'step {n}', 'vector (cr_step_symbolic) vs the symbolic-only env',
                 vec.cpu().numpy().view(np.uint32), only_vec.view(np.uint32))
  print('launches per step by kind (0 rgb, 1 semantic, 2 symbolic):', sorted(set(launches)))
  env.close()
  only.close()
  sym = crafter_b200.Env(num_envs=4, seed=1, observation='symbolic')
  sym.reset()
  pinned = [torch.zeros(4, dtype=d).pin_memory() for d in (torch.int32, torch.float32, torch.bool)]
  with pytest.raises(RuntimeError, match="not available with observation='symbolic'"):
    sym.step_host(*pinned)
  with pytest.raises(ValueError, match='image'):
    crafter_b200.recorder.EpisodeRecorder(sym, '/nonexistent-not-created')
  sym.close()


def test_vector_env_symbolic_spaces_and_final_obs():
  import torch
  from crafter_b200 import vector
  B, length, grid = 8, 3, grid_of((9, 9))
  dim = symbolic_layout(grid)['daylight'].stop
  venv = vector.make('CrafterReward-v1', num_envs=B, seed=0, length=length, observation='symbolic')
  assert tuple(venv.single_observation_space.shape) == (dim,) and tuple(venv.observation_space.shape) == (B, dim)
  assert venv.single_observation_space.dtype == np.float32 and float(np.max(venv.single_observation_space.high)) == 1
  oracle = oracle_env.OracleBatch(B, seed=0, length=length)
  everyone = np.arange(B)
  obs, _ = venv.reset()
  oracle.reset(render=False)
  check_vectors('vector reset', 'vector', obs.cpu().numpy(), oracle_vectors(oracle, grid, everyone), everyone, grid)
  finals = 0
  for n in range(2 * length):
    actions = np.full(B, 0, np.int32)
    obs, reward, terminated, truncated, info = venv.step(torch.from_numpy(actions).to(venv.env.device))
    _, _, ref_done = oracle.step(actions, auto_reset=False, render=False)
    ended = np.flatnonzero(ref_done)
    if len(ended):
      check_vectors(f'vector step {n}', 'final_obs', info['final_obs'].cpu().numpy()[ended],
                    oracle_vectors(oracle, grid, ended), ended, grid)
      assert info['_final_obs'].cpu().numpy()[ended].all()
      finals += len(ended)
      oracle.reset(ended, render=False)
    check_vectors(f'vector step {n}', 'vector', obs.cpu().numpy(), oracle_vectors(oracle, grid, everyone), everyone,
                  grid)
  assert finals == 2 * B
  venv.close()
