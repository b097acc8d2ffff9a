"""`-m gpu`: levels (Env.set_levels, Env.reset(mask, levels)) on the H100 against OracleBatch with levels
(tests/oracle_levels.LevelBatch), bit for bit, with the output buffers poisoned before every step (tests/test_full_batch_gpu.py).

* The benchmarked default workload at B = 4096 with auto-reset for 1,300 steps in the level-replay (PLR) pattern:
  after every step the envs that finished get levels drawn from a set of 200 world seeds (and now and then -1),
  through set_levels (the next episode plays them) or, on a tenth of the steps, reset(done, levels) (the episode
  that auto-reset just started is replaced at once).  Every step: done, reward, the player vector, the step
  counter, info['world_seed'], info['final_world_seed'] of the finished envs, the terminal frames, and the frames
  of a sample of envs; at checkpoints every env's canonical state and frame.
* Two sweep geometries at B = 8 * num_sms + 1 across nightfall, the same pattern.
* Envs on one level fed the same actions draw identical frames.
* The plumbing of the public interface: state_dict round trip with levels, an older snapshot without them, the
  checks of set_levels, cr_set_levels on a handle without a level buffer, the vector env's options['levels']."""
import time

import numpy as np
import pytest

import bench
from crafter_b200 import state as state_lib
from oracle import canon
from oracle import oracle_env
from tests import geometry_cases as gc
from tests import oracle_levels
from tests.parity import POISON, frame_problem
from tests.test_full_batch_gpu import PLAYER_FIELDS, check_frames, check_rows, gpu_canonical, gpu_player

pytestmark = pytest.mark.gpu

PS = state_lib.PS
SEED = 0
SAMPLE = 512


def level_pool(n=200, seed=7):
  rs = np.random.RandomState(seed)
  return np.concatenate([[0, 2 ** 31 - 2], rs.randint(0, 2 ** 31 - 1, n - 2)]).astype(np.int32)


def run_plr(B, steps, geometry, length=10000, checkpoints=(), reset_every=10, final_obs=True):
  """The PLR pattern on Env against OracleBatch; returns what the run reached."""
  import torch
  import crafter_b200
  env = crafter_b200.Env(num_envs=B, seed=SEED, auto_reset=True, length=length, final_obs=final_obs, **geometry)
  oracle = oracle_levels.LevelBatch(B, seed=SEED, length=length, **geometry)
  dev = env.device
  pool = level_pool()
  rs, pick = np.random.RandomState(SEED), np.random.RandomState(1)
  sample = np.sort(np.concatenate([[0, B - 1], 1 + np.random.RandomState(2).choice(B - 2, min(SAMPLE, B) - 2,
                                                                                  replace=False)]))
  sample_t = torch.as_tensor(sample, device=dev)
  episode = np.ones(B, np.int64)
  level = np.full(B, -1, np.int64)
  ws = np.array([oracle_env.world_seed(SEED + i, 1) for i in range(B)], np.int64)

  def start(ids):  # the oracle side of an episode start in the envs `ids`
    oracle.reset(ids, render=False)
    for i in ids:
      episode[i] += 1
      ws[i] = level[i] if level[i] >= 0 else oracle_env.world_seed(SEED + i, int(episode[i]))

  def poison():
    with torch.cuda.stream(env._stream):
      env._obs.fill_(POISON)
      if final_obs:
        env._final_obs.fill_(POISON)
      env._state['final_world_seed'].fill_(-7)

  def checkpoint(where, obs):
    arrays = {k: env.state[k].cpu().numpy() for k in ('mat', 'ents', 'inventory', 'achievements', 'pstate', 'touched')}
    for i in range(B):
      problem = canon.diff(oracle.envs[i].export_state(), gpu_canonical(env, i, arrays))
      assert problem is None, f'{where} env {i} state (oracle vs GPU): {problem}'
    check_frames(where, 'obs', obs.cpu().numpy(), oracle.render(), range(B))

  poison()
  obs = env.reset()
  oracle.reset(render=False)
  checkpoint('reset', obs)
  age = np.zeros(B, np.int64)
  day = oracle_env.daylight_table(steps + 2)
  reached = dict(resets=0, relevelled=0, reset_calls=0, night=0.0, played=set())
  for n in range(1, steps + 1):
    where = f'step {n}'
    actions = rs.randint(0, 17, B).astype(np.int32)
    poison()
    obs, reward, done, info = env.step(torch.from_numpy(actions).to(dev))
    reward, done_np = reward.cpu().numpy(), done.cpu().numpy()
    _, ref_reward, ref_done = oracle.step(actions, auto_reset=False, render=False)
    age += 1
    check_rows(where, 'done', done_np, ref_done)
    check_rows(where, 'reward', reward, ref_reward.astype(np.float32))
    ended = np.flatnonzero(ref_done)
    if len(ended):
      ended_t = torch.as_tensor(ended, device=dev)
      check_rows(where, 'final_world_seed', info['final_world_seed'][ended_t].cpu().numpy(), ws[ended].astype(np.int32),
                 ended)
      if final_obs:
        check_frames(where, 'final_observation', info['final_observation'][ended_t].cpu().numpy(),
                     oracle.render(ended), ended)
      reached['played'] |= set(ws[ended].tolist())
      start(ended)  # the auto-reset inside the step
      age[ended] = 0
      reached['resets'] += len(ended)
      new = pool[pick.randint(0, len(pool), B)]
      new[pick.rand(B) < 0.05] = -1
      mask = np.zeros(B, bool)
      mask[ended] = True
      level[ended] = new[ended]
      oracle.set_levels(new[ended], ended)
      reached['relevelled'] += len(ended)
      if n % reset_every == 0:  # this episode starts now: its world is generated again for the new level
        obs = env.reset(torch.from_numpy(mask).to(dev), torch.from_numpy(new).to(dev))
        start(ended)
        reached['reset_calls'] += 1
      else:  # the next episode plays it
        env.set_levels(torch.from_numpy(new).to(dev), torch.from_numpy(mask).to(dev))
    check_rows(where, 'levels', env.levels.cpu().numpy(), level.astype(np.int32))
    got_player, ps = gpu_player(env)
    check_rows(where, 'player', got_player, oracle.player(), fields=PLAYER_FIELDS)
    check_rows(where, 'step counter', ps[:, PS['step']], age)
    check_rows(where, 'world_seed', ps[:, PS['world_seed']], ws.astype(np.int32))
    reached['night'] = max(reached['night'], float((day[np.minimum(age, steps)] < 0.5).mean()))
    if n in checkpoints:
      checkpoint(where, obs)
    else:
      check_frames(where, 'obs', obs[sample_t].cpu().numpy(), oracle.render(sample), sample)
  env.check_errors()
  env.close()
  return reached


def test_plr_pattern_at_the_benchmarked_batch():
  """The default workload at B = 4096, 1,300 steps (about 6 minutes on an H100, most of it the oracle)."""
  import torch
  cfg = bench.env_kwargs(bench.CONFIGS['default'])
  geometry = {k: cfg[k] for k in ('area', 'view', 'size')}
  t0 = time.perf_counter()
  reached = run_plr(cfg['num_envs'], 1300, geometry, checkpoints={10, 300, 1000, 1300})
  print(f'plr B={cfg["num_envs"]}: {reached["resets"]} episodes ended, {reached["reset_calls"]} reset(done, levels) '
        f'calls, {len(reached["played"])} world seeds played, max night fraction {reached["night"]:.2f}, '
        f'{time.perf_counter() - t0:.0f} s on {torch.cuda.get_device_name()}')
  assert reached['resets'] >= 3 * cfg['num_envs'] and reached['reset_calls'] >= 10
  assert {0, 2 ** 31 - 2} <= reached['played'] and len(reached['played'] & set(level_pool().tolist())) >= 150
  assert reached['night'] >= 0.5


@pytest.mark.parametrize('name', ['odd_geometry', 'view5x7'])
def test_plr_pattern_at_sweep_geometries_across_nightfall(name):
  import torch
  B = 8 * torch.cuda.get_device_properties(0).multi_processor_count + 1
  reached = run_plr(B, 220, gc.kwargs(name), length=190, checkpoints={190, 220}, reset_every=4)
  assert reached['resets'] >= B and reached['night'] >= 0.5, reached


def test_envs_on_one_level_draw_identical_frames():
  import torch
  import crafter_b200
  B, level = 64, 987654
  env = crafter_b200.Env(num_envs=B, seed=3, auto_reset=True, length=60)
  ref = oracle_levels.LevelEnv(seed=99, length=60)
  ref.set_level(level)
  obs = env.reset(levels=np.full(B, level, np.int32)).cpu().numpy()
  want = ref.reset()
  rs = np.random.RandomState(4)
  for t in range(150):
    assert (obs == obs[0]).all(), (t, 'frames of one level differ')
    assert frame_problem(obs[0], want) is None, (t, frame_problem(obs[0], want))
    a = int(rs.randint(0, 17))
    obs, reward, done, info = env.step(torch.full((B,), a, dtype=torch.int32, device=env.device))
    obs = obs.cpu().numpy()
    want, r, d = ref.step(a)
    if d:
      assert (info['final_world_seed'].cpu().numpy() == level).all()
      want = ref.reset()
    assert (info['world_seed'].cpu().numpy() == level).all()


def test_state_dict_and_errors_of_the_public_interface():
  import torch
  import crafter_b200
  from crafter_b200 import _cabi, vector
  env = crafter_b200.Env(num_envs=4, seed=5, auto_reset=True, length=5)
  env.reset(levels=np.array([11, -1, 12, -1], np.int32))
  assert env.levels.tolist() == [11, -1, 12, -1]
  saved = env.state_dict()
  assert saved['level'].tolist() == [11, -1, 12, -1] and 'final_world_seed' in saved
  for _ in range(7):
    env.step(torch.zeros(4, dtype=torch.int32))
  played = env.state['pstate'][:, PS['world_seed']].tolist()
  env.load_state_dict(saved)
  for _ in range(7):
    env.step(torch.zeros(4, dtype=torch.int32))
  assert env.state['pstate'][:, PS['world_seed']].tolist() == played and played[0] == 11 and played[2] == 12
  old = {k: v for k, v in saved.items() if k not in ('level', 'final_world_seed')}
  env.load_state_dict(old)  # a snapshot taken before levels existed: every env on the reference's sequence
  assert env.levels.tolist() == [-1] * 4
  for bad, match in ((np.array([0, 0, 0, 2 ** 31 - 1], np.int64), 'world seeds'), (np.zeros(3, np.int32), 'shape'),
                     (np.zeros(4, np.float32), 'integers'), (torch.full((4,), -2, dtype=torch.int32, device='cuda'),
                                                            'world seeds')):
    with pytest.raises(ValueError, match=match):
      env.set_levels(bad)
  assert env.levels.tolist() == [-1] * 4
  # cr_set_levels on a handle whose cr_state.level is NULL
  level = env._state.pop('level')
  try:
    handle, _ = env._create(tuple(int(v) for v in env._size))
  finally:
    env._state['level'] = level
  lib = _cabi.load()
  rc = lib.cr_set_levels(handle, None, env._level_in.data_ptr(), None)
  assert rc != 0 and b'no level buffer' in lib.cr_last_error()
  lib.cr_destroy(handle)
  venv = vector.VectorEnv(num_envs=4, seed=5, length=5)
  venv.reset(options={'levels': np.array([3, 3, -1, 3], np.int32)})
  assert venv.env.levels.tolist() == [3, 3, -1, 3]
  assert venv.env.state['pstate'][:, PS['world_seed']].tolist()[:2] == [3, 3]
  venv.set_levels(np.array([-1, 8, 8, 8], np.int32), mask=np.array([1, 0, 0, 1], bool))
  assert venv.env.levels.tolist() == [-1, 3, -1, 8]
  venv.close()
  env.close()
